"""CPU: the premise of the DiT's collapsed unconditional branch (Hunyuan3DDiT.forward, uncond_txt_shared), checked on the
fp32 oracle restatement (oracle/hy3d_ref.py): with an all-zero unconditional context and the same t for both samples,
the unconditional sample's text rows stay equal to each other after every double and single block."""
import os

import numpy as np
import torch

import hy3d_ref as R


def test_uncond_text_rows_stay_equal_through_every_block(golden_dir):
    z = np.load(os.path.join(golden_dir, "dit_mini.npz"))
    sd = {k[2:]: torch.from_numpy(z[k].astype(np.float32)) for k in z.files if k.startswith("w:")}
    x = torch.from_numpy(z["x"]).float()[:1].repeat(2, 1, 1)
    c = torch.from_numpy(z["cond"]).float()[:1]
    Lt = c.shape[1]
    cond = torch.cat([torch.randn(c.shape, generator=torch.Generator().manual_seed(0)), torch.zeros_like(c)])
    t = torch.full((2,), 0.37)
    taps = []
    R.dit_forward(sd, x, t, cond, int(z["cfg_heads"]), int(z["cfg_depth"]), int(z["cfg_depth_single"]), taps=taps)
    assert len(taps) == int(z["cfg_depth"]) + int(z["cfg_depth_single"])
    for i, tp in enumerate(taps):
        un = tp[1, :Lt]
        rel = ((un - un[:1]).norm() / un.norm()).item()
        assert rel <= 1e-6, f"block {i}: uncond text rows differ, rel {rel:.2e}"
        # the conditional sample's text rows are not equal: the check has something to tell apart
        co = tp[0, :Lt]
        assert ((co - co[:1]).norm() / co.norm()).item() > 1e-2
