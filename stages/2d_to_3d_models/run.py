#!/usr/bin/env python
"""Stage 3 (`python run.py -p 3`) on the r3g hot path: drop-in for src/2d_to_3d_models/run.py.

Contract kept (SURVEY.md section 8b.1): `--config <yaml>`; reads `prepped_for_hunyuan` if `use_banana` else
`input_folder_hy`; skips names containing wall/room/ceiling/floor; clears and writes
`output_folder_hy/<stem>/<stem>.glb`; config keys num_inf_steps_hy, octree_resolution_hy, num_chunks_hy, seed,
mini, use_all_available_cuda; non-zero exit on failure.

Differences, all on purpose:
  * one process per GPU (torchrun / torch.distributed, NCCL) instead of a spawn-pool that reloads both models for
    every image (reference run.py:108-133): each rank loads the weights once, takes images i % world == rank of
    the SORTED list, and the finished meshes are gathered to rank 0 (r3g/dist.py::MeshBatchGatherer, over NCCL
    when there is more than one rank), which writes each .glb as its mesh lands;
  * FloaterRemover runs on the GPU (r3g/postprocessors.py: union-find components, MeshLab's 0.5 % rule) and
    DegenerateFaceRemover is the reference's no-op round trip; FaceReducer (pymeshlab quadric decimation to 40 000 faces)
    and the texture pipeline are not mirrored (SURVEY.md section 8f rows 2 and 4) -- the .glb holds the cleaned,
    undecimated, untextured shape;
  * `--random-weights` builds the Hunyuan3D-2 architecture with seeded random weights when no checkpoint is
    reachable (this build environment has no network).

Launch:  python stages/2d_to_3d_models/run.py --config src/config.yaml
   or:   python -m torch.distributed.run --nproc-per-node 8 stages/2d_to_3d_models/run.py --config ...
"""
import argparse
import os
import shutil
import sys
import time

import torch
import torch.distributed as dist
import yaml
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))

from r3g.dist import MeshBatchGatherer, shard_indices  # noqa: E402
from r3g.pipelines import Hunyuan3DDiTFlowMatchingPipeline, SimpleMesh  # noqa: E402
from r3g.postprocessors import DegenerateFaceRemover, FloaterRemover  # noqa: E402


def load_config(path):
    """src/utils/global_utils.py:464-476."""
    with open(path) as fh:
        return yaml.safe_load(fh)


def clear_output_directory(path):
    """src/utils/global_utils.py:443-461: empty the directory, keep the directory."""
    for name in os.listdir(path):
        p = os.path.join(path, name)
        shutil.rmtree(p) if os.path.isdir(p) else os.remove(p)


def main():
    ap = argparse.ArgumentParser(description="Run 2D to 3D model generation.")
    ap.add_argument("--config", default="../src/config.yaml", type=str)
    ap.add_argument("--random-weights", action="store_true")
    args = ap.parse_args()
    config = load_config(args.config)

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))

    input_folder = config["prepped_for_hunyuan"] if config.get("use_banana") else config["input_folder_hy"]
    output_folder = config["output_folder_hy"]
    if rank == 0:
        os.makedirs(output_folder, exist_ok=True)
        clear_output_directory(output_folder)
    skip = ("wall", "walls", "room", "ceiling", "floor")
    names = sorted(f for f in os.listdir(input_folder)
                   if f.lower().endswith((".png", ".jpg", ".jpeg")) and not any(s in f.lower() for s in skip))
    if not names:
        raise FileNotFoundError(f"No images found in the input folder '{input_folder}'.")

    if args.random_weights:
        pipe = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=0, device=f"cuda:{local}")
    else:
        mini = config.get("mini", True)
        repo = "tencent/Hunyuan3D-2mini" if mini else "tencent/Hunyuan3D-2"
        kw = dict(subfolder="hunyuan3d-dit-v2-mini", variant="fp16") if mini else {}
        pipe = Hunyuan3DDiTFlowMatchingPipeline.from_pretrained(repo, device=f"cuda:{local}", **kw)
    pipe.vae.surface_extractor.keep_on_device = True     # the mesh leaves the GPU once, after the floater removal

    mine = shard_indices(len(names), rank, world)
    local_meshes, local_names = [], []
    for i in mine:
        t0 = time.time()
        image = Image.open(os.path.join(input_folder, names[i])).convert("RGBA")
        out = pipe(image=image, num_inference_steps=config.get("num_inf_steps_hy", 100),
                   octree_resolution=config.get("octree_resolution_hy", 380),
                   num_chunks=config.get("num_chunks_hy", 20000),
                   generator=torch.manual_seed(config.get("seed", 12345)), output_type="mesh")[0]
        stem = os.path.splitext(names[i])[0]
        if out is None:
            print(f"[rank {rank}] {stem}: no surface", flush=True)
            continue
        v, f = out.mesh_v, out.mesh_f
        if not torch.is_tensor(v):
            v, f = torch.from_numpy(v), torch.from_numpy(f)
        # src/2d_to_3d_models/run.py:93-94 (FaceReducer, :95, is not mirrored)
        v, f = DegenerateFaceRemover()(FloaterRemover()((v, f), device=f"cuda:{local}"))
        local_meshes.append((v, f))
        local_names.append(stem)
        print(f"[rank {rank}] {stem}: {v.shape[0]} vertices, {f.shape[0]} faces in {time.time() - t0:.2f} s", flush=True)

    all_names = [local_names]
    if world > 1:
        all_names = [None] * world
        dist.all_gather_object(all_names, local_names)
    gatherer = MeshBatchGatherer(max((v.shape[0] for v, _ in local_meshes), default=0),
                                 max((f.shape[0] for _, f in local_meshes), default=0),
                                 len(local_meshes), f"cuda:{local}", to_host=True)
    for v, f in local_meshes:
        gatherer.submit(v, f)
    written = []

    def write(k, r, v, f):              # v, f are views into the landing ring: used here, not kept
        stem = all_names[r][k]
        out_dir = os.path.join(output_folder, stem)
        os.makedirs(out_dir, exist_ok=True)
        # export_to_trimesh's winding flip (pipelines.py:102)
        SimpleMesh(v.numpy(), f.numpy()[:, ::-1]).export(os.path.join(out_dir, f"{stem}.glb"))
        written.append(stem)
    gatherer.finish(to_host=True, sink=write)
    if rank == 0:
        print(f"wrote {len(written)} mesh(es) to {output_folder}")
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
