"""GPU: one object on an object group (r3g/dist.py) is the single-GPU object bit for bit -- the lone-sample DiT forwards
against the CFG pair's B = 2 forward, the chunk-range decode against the whole decode, and the pipeline on a group of 2
(and 4) ranks against the same call without a group.  Run as a script under torch.distributed.run, this file is the
worker of the multi-rank tests."""
import json
import os
import signal
import socket
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))

pytestmark = pytest.mark.gpu

MINI = dict(
    model=dict(in_channels=64, context_in_dim=96, hidden_size=128, num_heads=2, depth=2, depth_single_blocks=2),
    vae=dict(num_latents=48, embed_dim=64, num_freqs=8, include_pi=False, heads=2, width=128, num_decoder_layers=2,
             qkv_bias=False, qk_norm=True, scale_factor=0.999),
    scheduler=dict(num_train_timesteps=1000),
    image_processor=dict(size=512, border_ratio=0.15),
)
MINI_DISTILLED = dict(MINI, model=dict(MINI["model"], guidance_embed=True),
                      scheduler=dict(target="hy3dgen.shapegen.schedulers.ConsistencyFlowMatchEulerDiscreteScheduler",
                                     num_train_timesteps=1000, pcm_timesteps=100))


# ------------------------------------------------------------------------------------------------ one device
def _run_forward(m, x, t, c, shared, graph):
    from r3g.graphs import GraphCache
    if not graph:
        return m(x, t, {"main": c}, uncond_txt_shared=shared).clone()
    g = GraphCache().get(0, (x, t, c), lambda xs, ts, cs: m(xs, ts, {"main": cs}, uncond_txt_shared=shared))
    g.replay()
    return g.outputs.clone()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("size", ["mini", "full_width_1_2"])
def test_lone_forwards_equal_the_cfg_pair(size, graph):
    """cond alone (B = 1, full path) and uncond alone (B = 1, collapsed to one text row) are the two halves of the
    collapsed B = 2 forward, torch.equal."""
    from r3g.dit import Hunyuan3DDiT
    if size == "mini":
        m, Li, Lt, C = Hunyuan3DDiT(**MINI["model"]).init_random(seed=3), 48, 24, 96
    else:
        m, Li, Lt, C = Hunyuan3DDiT(depth=1, depth_single_blocks=2).init_random(seed=4), 3072, 1370, 1536
    gen = torch.Generator(device="cuda").manual_seed(0)
    x1 = torch.randn(1, Li, 64, device="cuda", generator=gen).half()
    x = torch.cat([x1, x1])
    c = torch.cat([torch.randn(1, Lt, C, device="cuda", generator=gen), torch.zeros(1, Lt, C, device="cuda")]).half()
    t = torch.tensor([0.3469, 0.3469], device="cuda").half()
    pair = _run_forward(m, x, t, c, True, graph)
    assert torch.equal(pair, _run_forward(m, x, t, c, False, graph))
    cond = _run_forward(m, x[:1], t[:1], c[:1].contiguous(), False, graph)
    unc = _run_forward(m, x[1:].contiguous(), t[1:].contiguous(), c[1:].contiguous(), True, graph)
    assert torch.equal(torch.cat([cond, unc]), pair)
    assert torch.equal(unc, _run_forward(m, x[1:].contiguous(), t[1:].contiguous(), c[1:].contiguous(), False, graph))


@pytest.fixture(scope="module")
def geo():
    from r3g.pipelines import HUNYUAN3D_2_CONFIG
    from r3g.vae import ShapeVAE
    return ShapeVAE(**HUNYUAN3D_2_CONFIG["vae"]).init_random(seed=5).geo_decoder


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("R,G", [(256, 4), (100, 3)])
def test_decode_by_chunk_ranges_stitches_to_the_whole_decode(geo, R, G, graph, monkeypatch):
    from r3g.dist import chunk_ranges
    monkeypatch.setattr(geo, "use_cuda_graph", graph)
    gen = torch.Generator(device="cuda").manual_seed(6)
    lat = (torch.randn(1, 3072, 1024, device="cuda", generator=gen) * 0.5).half()
    bounds = [-1.01] * 3 + [1.01] * 3
    full = torch.empty(R + 1, R + 1, R + 1, device="cuda")
    geo.decode_grid(lat, bounds, R, full)
    stitched = torch.full_like(full, float("nan"))
    n_chunks = geo.grid_chunks(R)[1]
    ranges = chunk_ranges(n_chunks, G)
    for c in ranges:
        part = torch.full_like(full, float("nan"))
        geo.decode_grid(lat, bounds, R, part, chunks=c)
        s0, s1 = geo.chunk_span(R, c)
        flat = part.view(-1)
        assert not flat[s0:s1].isnan().any() and flat[:s0].isnan().all() and flat[s1:].isnan().all()
        stitched.view(-1)[s0:s1] = flat[s0:s1]
    assert torch.equal(stitched, full)


def test_decode_graphs_of_every_chunk_range_stay_cached():
    """A rank that alternates whole objects with its shares of split ones (G = 2, 4, 8 as member 0 or 1) captures each
    decode graph once and replays it afterwards; another grid geometry drops them."""
    from r3g.dist import chunk_ranges
    from r3g.pipelines import HUNYUAN3D_2_CONFIG
    from r3g.vae import ShapeVAE
    cfg = dict(HUNYUAN3D_2_CONFIG["vae"], width=128, heads=2, num_decoder_layers=1)
    geo = ShapeVAE(**cfg).init_random(seed=8).geo_decoder
    lat = (torch.randn(1, 3072, 128, device="cuda", generator=torch.Generator(device="cuda").manual_seed(9)) * 0.5).half()
    bounds = [-1.01] * 3 + [1.01] * 3
    R = 128
    n = geo.grid_chunks(R)[1]
    arms = [None] + [chunk_ranges(n, G)[m] for G in (2, 4, 8) for m in (0, 1)]
    grids = {}
    for rnd in range(3):
        for c in arms:
            out = torch.full((R + 1,) * 3, float("nan"), device="cuda")
            geo.decode_grid(lat, bounds, R, out, chunks=c)
            s0, s1 = geo.chunk_span(R, c)
            if rnd == 0:
                grids[c] = out.view(-1)[s0:s1].clone()
            else:
                assert torch.equal(out.view(-1)[s0:s1], grids[c])
        if rnd == 0:
            captured = geo._graphs.captures
            assert captured == len(arms) == len(geo._graphs.entries)
    assert geo._graphs.captures == captured                     # rounds 1 and 2 replayed every graph
    geo.decode_grid(lat, bounds, R - 1, torch.empty((R,) * 3, device="cuda"))
    assert len(geo._graphs.entries) == 1                        # another geometry: one graph again


# ------------------------------------------------------------------------------------------------ several ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _launch(nproc, out, backend, timeout=900):
    """torch.distributed.run of this file at world size nproc; the whole process group is killed on a timeout."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.abspath(__file__), "--out", str(out), "--backend", backend]
    p = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, start_new_session=True)
    try:
        log, _ = p.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)
        log, _ = p.communicate()
        raise AssertionError(f"world of {nproc} timed out:\n{log[-3000:]}")
    assert p.returncode == 0, log[-3000:]
    return [json.load(open(os.path.join(out, f"rank{r}.json"))) for r in range(nproc)]


def _check_group_results(res):
    for r, rr in enumerate(res):
        for case, got in rr.items():
            if case == "mismatched_seed":
                assert got == "raised", (r, case, got)
            elif r == 0:
                assert got["grid_equal"] and got["mesh_equal"] and got["faces"] > 0, (case, got)
            else:
                assert got == "none", (r, case, got)


@pytest.mark.parametrize("world", [2, 4])
def test_pipeline_on_a_group_nccl(world, tmp_path):
    """One NCCL rank per GPU: the leader's grid and mesh equal the same call without a group (base CFG, distilled)."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    _check_group_results(_launch(world, tmp_path, "nccl"))


def test_pipeline_on_a_group_sharing_one_gpu(tmp_path):
    """Two gloo ranks on one GPU (gloo stages the CUDA tensors through the host): the same checks as on NCCL, so that
    the group path runs on a one-GPU machine too."""
    _check_group_results(_launch(2, tmp_path, "gloo"))


def test_stage3_twin_splits_the_tail_object(tmp_path):
    """3 images on 2 ranks: objects 0 and 1 one per rank, object 2 on both; the .glb files are byte-identical to a
    one-rank run."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import yaml
    from PIL import Image
    inp = tmp_path / "in"
    inp.mkdir()
    import numpy as np
    rng = np.random.default_rng(0)
    for i in range(3):
        a = np.zeros((256, 256, 4), np.uint8)
        a[64:192, 48 + 8 * i:208, :3] = rng.integers(0, 255, (128, 160 - 8 * i, 3))
        a[64:192, 48 + 8 * i:208, 3] = 255
        Image.fromarray(a).save(inp / f"obj{i}.png")
    outs = {}
    for world in (1, 2):
        out = tmp_path / f"out{world}"
        out.mkdir()
        cfg = dict(use_banana=False, input_folder_hy=str(inp), output_folder_hy=str(out), num_inf_steps_hy=3,
                   octree_resolution_hy=128, num_chunks_hy=16000, seed=1234567, mini=False)
        (tmp_path / f"config{world}.yaml").write_text(yaml.safe_dump(cfg))
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", str(world), "--master-addr",
               "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "stages", "2d_to_3d_models", "run.py"),
               "--config", str(tmp_path / f"config{world}.yaml"), "--random-weights"]
        p = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, start_new_session=True)
        try:
            log, _ = p.communicate(timeout=1200)
        except subprocess.TimeoutExpired:
            os.killpg(p.pid, signal.SIGKILL)
            p.communicate()
            raise
        assert p.returncode == 0, log[-3000:]
        outs[world] = {f"obj{i}": (out / f"obj{i}" / f"obj{i}.glb").read_bytes() for i in range(3)}
    assert outs[1] == outs[2]


# ------------------------------------------------------------------------------------------------ worker
def _worker(out, backend):
    import numpy as np
    import torch.distributed as dist
    from r3g.pipelines import Hunyuan3DDiTFlowMatchingPipeline
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]) if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, **({"device_id": dev} if backend == "nccl" else {}))
    group = dist.new_group(list(range(world)))
    res = {}
    try:
        # flashvdm_cfg: the decode is not split, the leader runs it alone
        for case, config, steps in (("base_cfg", MINI, 6), ("distilled", MINI_DISTILLED, 5), ("flashvdm_cfg", MINI, 6)):
            pipe = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=11, config=config, conditioner=None, device=dev)
            if case == "flashvdm_cfg":
                pipe.enable_flashvdm()
            torch.manual_seed(0)
            cfg = case != "distilled"
            main = torch.randn(1, 24, 96)
            cond = {"main": (torch.cat([main, torch.zeros(1, 24, 96)]) if cfg else main).to(dev).half()}
            kw = dict(cond=cond, num_inference_steps=steps, guidance_scale=5.0, octree_resolution=64,
                      output_type="mesh", enable_pbar=False)
            # the call without a group, on every rank; the iso level is the grid's median (FlashVDM: of the evaluated
            # points), so that random weights give a surface
            pipe(generator=torch.manual_seed(1234567), **kw)
            ref_grid = pipe.last_grid.clone()
            level = float(ref_grid.float().nanmedian())
            ref = pipe.vae.surface_extractor(ref_grid, mc_level=level, bounds=1.01, octree_resolution=64)[0]
            got = pipe(generator=torch.manual_seed(1234567), object_group=group, mc_level=level, **kw)
            if rank != 0:
                res[case] = "none" if got == [None] else "mesh"
                continue
            got = got[0]
            grid = pipe.last_grid
            same = (grid == ref_grid) | (grid.isnan() & ref_grid.isnan())      # FlashVDM: NaN where not evaluated
            res[case] = dict(grid_equal=bool(grid.shape == ref_grid.shape and same.all()), faces=int(len(ref.mesh_f)),
                             mesh_equal=bool(np.array_equal(got.mesh_v, ref.mesh_v)
                                             and np.array_equal(got.mesh_f, ref.mesh_f)))
        try:        # member 1 draws other initial latents: every member must raise
            pipe(generator=torch.manual_seed(1234567 + (rank == 1)), object_group=group, **kw)
            res["mismatched_seed"] = "returned"
        except RuntimeError:
            res["mismatched_seed"] = "raised"
        with open(os.path.join(out, f"rank{rank}.json"), "w") as fh:
            json.dump(res, fh)
        dist.barrier()
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--backend", default="nccl")
    a = ap.parse_args()
    _worker(a.out, a.backend)
