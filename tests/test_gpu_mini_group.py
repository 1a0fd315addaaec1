"""GPU: Hunyuan3D-2mini's denoiser (HunYuanDiTPlain) on an object group -- two gloo ranks sharing one GPU give the
single-GPU grid and mesh bit for bit (the CFG pair split over the members, _denoise_group with the context k / v
projected once per call)."""
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

MINI_PLAIN = dict(
    model=dict(target="hy3dgen.shapegen.models.denoisers.hunyuandit.HunYuanDiTPlain", in_channels=64, hidden_size=128,
               context_dim=96, depth=5, num_heads=2, qk_norm=True, use_attention_pooling=False, qkv_bias=False,
               num_moe_layers=2, num_experts=4, moe_top_k=2),
    vae=dict(num_latents=48, embed_dim=64, num_freqs=8, include_pi=False, heads=2, width=128, num_decoder_layers=2,
             qkv_bias=False, qk_norm=True, scale_factor=0.999),
    scheduler=dict(num_train_timesteps=1000),
    image_processor=dict(size=512, border_ratio=0.15),
)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.gpu
def test_2mini_on_two_gloo_ranks_equals_one_gpu(tmp_path):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.abspath(__file__), "--out", str(tmp_path)]
    p = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, start_new_session=True)
    try:
        log, _ = p.communicate(timeout=600)
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)
        log, _ = p.communicate()
        raise AssertionError(f"timed out:\n{log[-3000:]}")
    assert p.returncode == 0, log[-3000:]
    res = [json.load(open(os.path.join(tmp_path, f"rank{r}.json"))) for r in range(2)]
    assert res[0]["grid_equal"] and res[0]["mesh_equal"] and res[0]["faces"] > 0, res[0]
    assert res[1] == {"got": "none"}


def _worker(out):
    import numpy as np
    import torch.distributed as dist
    from r3g.dit_plain import HunYuanDiTPlain
    from r3g.pipelines import Hunyuan3DDiTFlowMatchingPipeline
    rank = int(os.environ["RANK"])
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo")
    group = dist.new_group([0, 1])
    try:
        pipe = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=11, config=MINI_PLAIN, conditioner=None, device=dev)
        assert isinstance(pipe.model, HunYuanDiTPlain)
        torch.manual_seed(0)
        main = torch.randn(1, 24, 96)
        cond = {"main": torch.cat([main, torch.zeros(1, 24, 96)]).to(dev).half()}
        kw = dict(cond=cond, num_inference_steps=6, guidance_scale=5.0, octree_resolution=64, output_type="mesh",
                  enable_pbar=False)
        pipe(generator=torch.manual_seed(1234567), **kw)
        ref_grid = pipe.last_grid.clone()
        level = float(ref_grid.float().nanmedian())
        ref = pipe.vae.surface_extractor(ref_grid, mc_level=level, bounds=1.01, octree_resolution=64)[0]
        got = pipe(generator=torch.manual_seed(1234567), object_group=group, mc_level=level, **kw)
        if rank != 0:
            res = {"got": "none" if got == [None] else "mesh"}
        else:
            got = got[0]
            res = dict(grid_equal=bool(torch.equal(pipe.last_grid, ref_grid)), faces=int(len(ref.mesh_f)),
                       mesh_equal=bool(np.array_equal(got.mesh_v, ref.mesh_v) and np.array_equal(got.mesh_f, ref.mesh_f)))
        with open(os.path.join(out, f"rank{rank}.json"), "w") as fh:
            json.dump(res, fh)
        dist.barrier()
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    _worker(ap.parse_args().out)
