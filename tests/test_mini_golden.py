"""CPU: the Hunyuan3D-2mini fixture (tests/golden/hunyuandit_plain_mini.npz, from the reference's own HunYuanDiTPlain and
MoEBlock by oracle/make_golden_mini.py) against the float32 restatement oracle/hy3d_mini_ref.py, on the fixture's own
gate routing, at odd and even depth; and the generator's reproducibility."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
FIXTURE = os.path.join(ROOT, "tests", "golden", "hunyuandit_plain_mini.npz")
BASE = dict(in_channels=64, hidden_size=128, context_dim=96, num_heads=2, qk_norm_type="rms", num_moe_layers=2,
            num_experts=4, moe_top_k=2)


def fixture_case(z, name):
    """(config, reference state dict, x, t, cond, gate routes) of one geometry of the fixture."""
    import hy3d_mini_ref as R
    sd = R.mini_state_dict(z[f"{name}_w_keys"], z[f"{name}_w_shapes"], int(z[f"{name}_w_seed"]))
    cfg = dict(BASE, depth=int(z[f"{name}_depth"]), qkv_bias=bool(z[f"{name}_qkv_bias"]))
    routes = [(torch.from_numpy(z[f"{name}_gate{i}_ids"]), torch.from_numpy(z[f"{name}_gate{i}_w"])) for i in range(2)]
    return (cfg, sd, torch.from_numpy(z[f"{name}_x"]), torch.from_numpy(z[f"{name}_t"]),
            torch.from_numpy(z[f"{name}_cond"]), routes)


@pytest.mark.parametrize("name", ["odd", "even"])
def test_fixture_matches_the_float32_oracle_per_block(name):
    import hy3d_mini_ref as R
    z = np.load(FIXTURE)
    cfg, sd, x, t, cond, routes = fixture_case(z, name)
    taps = []
    with torch.no_grad():
        y = R.forward(sd, cfg, x, t, cond, routes=routes, taps=taps)
    assert len(taps) == cfg["depth"]
    for i, tp in enumerate(taps):
        ref = torch.from_numpy(z[f"{name}_tap{i}"])
        assert (tp - ref).abs().max() <= 1e-4 * ref.abs().max(), (name, i)
    ref = torch.from_numpy(z[f"{name}_y"])
    assert (y - ref).abs().max() <= 1e-4 * ref.abs().max()
    # every row of both MoE blocks was routed to two distinct experts
    for ids, w in routes:
        assert ids.shape == (2 * 41, 2) and (ids[:, 0] != ids[:, 1]).all() and (w > 0).all()


def test_generator_reproduces_the_fixture(tmp_path):
    import ref_import
    if not ref_import.available():
        pytest.skip("the reference checkout is not present")
    import make_golden_mini
    d = make_golden_mini.generate(str(tmp_path / "mini.npz"))
    z = np.load(FIXTURE)
    assert sorted(d) == sorted(z.files)
    for k in z.files:
        assert np.array_equal(d[k], z[k]), k
