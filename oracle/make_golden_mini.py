#!/usr/bin/env python
"""ORACLE -- test infrastructure only.

Generates tests/golden/hunyuandit_plain_mini.npz by running the REFERENCE's own HunYuanDiTPlain and MoEBlock
(Hunyuan3D-2/hy3dgen/shapegen/models/denoisers/hunyuandit.py, moe_layers.py) in float32 on the CPU.  Run in the build
container only:
    python oracle/make_golden_mini.py

moe_layers.py imports diffusers' FeedForward, which is not installed here.  The stand-in below has diffusers' module
tree and therefore its state-dict keys (net.0.proj, net.2) and computes what FeedForward(dim, activation_fn="gelu",
inner_dim, bias=True, dropout=0, final_dropout=False) computes in eval mode: Linear, erf-GELU, Dropout(0), Linear.

Two geometries, head_dim 64, E = 4 experts, top-2: depth 5 (odd; every pushed state is popped) with qkv_bias, and
depth 6 (even; block 0's pushed state is never used) without.  Both have 2 MoE blocks.  Stored per geometry: the
weights as key names, shapes and a seed (hy3d_mini_ref.mini_state_dict regenerates them), the fp16-valued inputs, the
hidden state after every block, each MoE gate's expert ids and weights, and the output.
"""
import importlib
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_import  # noqa: E402
import hy3d_mini_ref as R  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "hunyuandit_plain_mini.npz")
GEOMETRIES = {"odd": dict(depth=5, qkv_bias=True, seed=11), "even": dict(depth=6, qkv_bias=False, seed=12)}
BASE = dict(input_size=40, in_channels=64, hidden_size=128, context_dim=96, num_heads=2, qk_norm=True,
            qk_norm_type="rms", text_len=24, use_attention_pooling=False, num_moe_layers=2, num_experts=4, moe_top_k=2)


class _GELU(nn.Module):          # diffusers.models.activations.GELU(dim_in, dim_out, approximate="none", bias=True)
    def __init__(self, dim_in, dim_out, bias=True):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out, bias=bias)

    def forward(self, x):
        return torch.nn.functional.gelu(self.proj(x))


class FeedForward(nn.Module):    # stand-in for diffusers.models.attention.FeedForward (see the module docstring)
    def __init__(self, dim, dim_out=None, mult=4, dropout=0.0, activation_fn="gelu", final_dropout=False,
                 inner_dim=None, bias=True):
        super().__init__()
        assert activation_fn == "gelu" and not final_dropout
        inner_dim = inner_dim or int(dim * mult)
        self.net = nn.ModuleList([_GELU(dim, inner_dim, bias), nn.Dropout(dropout), nn.Linear(inner_dim, dim_out or dim,
                                                                                             bias=bias)])

    def forward(self, x):
        for m in self.net:
            x = m(x)
        return x


def reference_module():
    if "diffusers.models.attention" not in sys.modules:
        for name in ("diffusers", "diffusers.models", "diffusers.models.attention"):
            sys.modules.setdefault(name, types.ModuleType(name))
        sys.modules["diffusers.models.attention"].FeedForward = FeedForward
    base = os.path.join(ref_import.HY, "hy3dgen")
    ref_import._stub_pkg("hy3dgen", base)
    ref_import._stub_pkg("hy3dgen.shapegen", os.path.join(base, "shapegen"))
    ref_import._stub_pkg("hy3dgen.shapegen.models", os.path.join(base, "shapegen/models"))
    ref_import._stub_pkg("hy3dgen.shapegen.models.denoisers", os.path.join(base, "shapegen/models/denoisers"))
    return importlib.import_module("hy3dgen.shapegen.models.denoisers.hunyuandit")


def golden(name, geo):
    m = reference_module()
    cfg = dict(BASE, depth=geo["depth"], qkv_bias=geo["qkv_bias"])
    model = m.HunYuanDiTPlain(**cfg).eval()
    keys = list(model.state_dict())
    shapes = [tuple(model.state_dict()[k].shape) for k in keys]
    model.load_state_dict(R.mini_state_dict(keys, shapes, geo["seed"]), strict=True)
    g = torch.Generator().manual_seed(geo["seed"])
    B, Li, Lt = 2, 40, 24
    x = torch.randn(B, Li, 64, generator=g).half().float()
    cond = torch.randn(B, Lt, 96, generator=g).half().float()
    t = torch.tensor([0.3469, 0.8125]).half().float()
    taps, gates = [], []
    hooks = [b.register_forward_hook(lambda mod, i, o: taps.append(o.detach().clone())) for b in model.blocks]
    hooks += [b.moe.gate.register_forward_hook(lambda mod, i, o: gates.append((o[0].clone(), o[1].clone())))
              for b in model.blocks if b.use_moe]
    with torch.no_grad():
        y = model(x, t, {"main": cond})
    for h in hooks:
        h.remove()
    width = max(len(s) for s in shapes)
    d = {f"{name}_w_keys": np.array(keys),
         f"{name}_w_shapes": np.array([list(s) + [0] * (width - len(s)) for s in shapes]),
         f"{name}_w_seed": np.int64(geo["seed"]), f"{name}_depth": np.int64(geo["depth"]),
         f"{name}_qkv_bias": np.int64(geo["qkv_bias"]),
         f"{name}_x": x.half().numpy(), f"{name}_t": t.half().numpy(), f"{name}_cond": cond.half().numpy(),
         f"{name}_y": y.numpy()}
    for i, tp in enumerate(taps):
        d[f"{name}_tap{i}"] = tp.numpy()
    for i, (ids, w) in enumerate(gates):
        d[f"{name}_gate{i}_ids"] = ids.numpy().astype(np.int32)
        d[f"{name}_gate{i}_w"] = w.numpy()
    return d


def generate(path=OUT):
    torch.set_num_threads(4)
    d = {}
    for name, geo in GEOMETRIES.items():
        d.update(golden(name, geo))
    np.savez_compressed(path, **d)
    return d


if __name__ == "__main__":
    assert ref_import.available(), "reference checkout not found"
    d = generate()
    print("hunyuandit_plain_mini:", {k: v.shape for k, v in d.items() if "tap" in k or k.endswith("_y")})
