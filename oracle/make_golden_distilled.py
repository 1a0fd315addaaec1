#!/usr/bin/env python
"""ORACLE -- test infrastructure only.

Generates the guidance-distilled fixtures under tests/golden/ by running the REFERENCE's own modules, like
make_golden.py (whose fixtures it leaves untouched).  Run in the build container only:
    python oracle/make_golden_distilled.py

  dit_guidance_mini.npz    Hunyuan3DDiT(guidance_embed=True) at make_golden.golden_dit's mini geometry, B = 2 with a
                           different guidance per sample, the per-block taps, and the reference timestep_embedding in
                           fp16 at guidance-sized arguments (1000 * guidance up to 10 000).  The weights are stored as
                           key names, shapes and a seed: hy3d_distilled_ref.mini_state_dict regenerates them.
  scheduler_consistency.npz  ConsistencyFlowMatchEulerDiscreteScheduler: timesteps, sigmas_ and step() outputs on fp16
                           inputs for N in {1, 2, 5, 8, 50} x pcm_timesteps in {50, 100}
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_import  # noqa: E402
import hy3d_distilled_ref as D  # noqa: E402
from make_golden import OUT  # noqa: E402

SEED = 6

STEPS = (1, 2, 5, 8, 50)
PCMS = (50, 100)
GUIDANCE_EMB = (1.0, 3.5, 5.0, 5.3, 7.5, 10.0)


def golden_dit_guidance():
    m = ref_import.hunyuan_dit()
    cfg = dict(in_channels=64, context_in_dim=96, hidden_size=128, num_heads=2, depth=2, depth_single_blocks=2,
               axes_dim=[64], guidance_embed=True)
    model = m.Hunyuan3DDiT(**cfg).eval()
    # the weights are not stored (they would be most of the file): the tests regenerate them from the keys and shapes
    keys = list(model.state_dict())
    shapes = [tuple(model.state_dict()[k].shape) for k in keys]
    model.load_state_dict(D.mini_state_dict(keys, shapes, SEED), strict=True)
    torch.manual_seed(6)
    B, L, Lc = 2, 40, 24
    x = torch.randn(B, L, 64).half().float()
    cond = torch.randn(B, Lc, 96).half().float()
    t = torch.tensor([0.3469, 0.3469]).half().float()
    # 1000 * g is exact in fp16 for both, so the fp32 module sees the values the fp16 pipeline does
    guidance = torch.tensor([3.5, 7.5])
    taps = []
    hooks = [blk.register_forward_hook(lambda mod, i, o: taps.append(
        torch.cat((o[1], o[0]), 1) if isinstance(o, tuple) else o)) for blk in
        list(model.double_blocks) + list(model.single_blocks)]
    with torch.no_grad():
        y = model(x, t, {"main": cond}, guidance=guidance)
        y_other = model(x, t, {"main": cond}, guidance=guidance.flip(0))
    for h in hooks:
        h.remove()
    width = max(len(s) for s in shapes)
    d = dict(w_keys=np.array(keys), w_shapes=np.array([list(s) + [0] * (width - len(s)) for s in shapes]),
             w_seed=np.int64(SEED))
    # x and cond are fp16 values: stored as fp16
    d.update(x=x.half().numpy(), t=t.numpy(), cond=cond.half().numpy(), guidance=guidance.numpy(), y=y.numpy(),
             y_flipped=y_other.numpy(), cfg_heads=np.int64(2), cfg_depth=np.int64(2), cfg_depth_single=np.int64(2))
    for i, tp in enumerate(taps[:4]):
        d[f"tap{i}"] = tp.numpy()
    g16 = torch.tensor(GUIDANCE_EMB, dtype=torch.float16)
    d["gemb_g"] = g16.numpy()
    d["gemb_out"] = m.timestep_embedding(g16, 256, 1000.0).numpy()   # positional max_period, hunyuan3ddit.py:396
    np.savez_compressed(os.path.join(OUT, "dit_guidance_mini.npz"), **d)
    print("dit_guidance_mini: y", tuple(y.shape), "taps", len(taps[:4]),
          "guidance swap changes y by", float((y - y_other).abs().max()))


def golden_scheduler_consistency():
    s = ref_import.hunyuan_scheduler()
    d = {}
    for pcm in PCMS:
        sch = s.ConsistencyFlowMatchEulerDiscreteScheduler(num_train_timesteps=1000, pcm_timesteps=pcm)
        d[f"table_{pcm}"] = sch.sigmas.numpy()
        for n in STEPS:
            sch.set_timesteps(sigmas=np.linspace(0, 1, n))
            d[f"timesteps_{n}_{pcm}"] = sch.timesteps.numpy()
            d[f"sigmas__{n}_{pcm}"] = sch.sigmas_.numpy()
            # every step of the schedule on fp16 inputs, the dtype flow of pipelines.py:755-756
            torch.manual_seed(1000 * pcm + n)
            x = torch.randn(1, 4, 64).half()
            xs, vs, preds = [x.numpy()], [], []
            for t in sch.timesteps:
                v = torch.randn(1, 4, 64).half()
                out = sch.step(v, t, x)
                x = out.prev_sample
                vs.append(v.numpy())
                xs.append(x.numpy())
                preds.append(out.pred_original_sample.numpy())
            d[f"x_{n}_{pcm}"], d[f"v_{n}_{pcm}"], d[f"pred_{n}_{pcm}"] = np.stack(xs), np.stack(vs), np.stack(preds)
    np.savez_compressed(os.path.join(OUT, "scheduler_consistency.npz"), **d)
    print("scheduler_consistency: sigmas_ N=5 pcm=100", d["sigmas__5_100"])


if __name__ == "__main__":
    assert ref_import.available(), "reference checkout not found"
    torch.set_num_threads(8)
    golden_dit_guidance()
    golden_scheduler_consistency()
