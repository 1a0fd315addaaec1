#!/usr/bin/env python
"""ORACLE -- fixture generator (needs the reference checkout, see oracle/ref_import.py).

Generates tests/golden/multiview.npz by running the REFERENCE's own multi-view classes (Hunyuan3D-2mv) on the inputs
that tests/test_multiview.py rebuilds from the functions below:

  proc_*        MVImageProcessorV2 (preprocessors.py:120-159) on seeded synthetic RGBA views, for every case of
                PROC_CASES (dict orders, subsets of 1-4 views, PIL and path inputs): view_idxs, shapes, dtypes and the
                sha256 of the image / mask tensors
  table_<C>     the view_embed table of DinoImageEncoderMV (get_1d_sincos_pos_embed_from_grid, conditioner.py:37-54)
                at C = 1536 and at the small test width, float32 [view_num, C]
  enc_*         DinoImageEncoderMV (conditioner.py:134-200) on the small ENC_CFG model with weights regenerated from
                ENC_SEED (enc_state_dict), for every case of ENC_CASES (B in {1, 2}, V in {1, 2, 4}, with and without
                view_idxs): outputs, and the unconditional embedding

    python oracle/make_golden_multiview.py
"""
import hashlib
import importlib.util
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import ref_import  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "multiview.npz")

TAGS = ("front", "left", "back", "right")

# (case name, view tags in dict order, "pil" or "path")
PROC_CASES = (
    ("all_sorted", ("front", "left", "back", "right"), "pil"),
    ("all_reversed", ("right", "back", "left", "front"), "pil"),
    ("all_shuffled", ("back", "front", "right", "left"), "path"),
    ("three", ("back", "front", "left"), "pil"),
    ("three_other_order", ("left", "back", "front"), "pil"),
    ("two", ("right", "front"), "path"),
    ("one_left", ("left",), "pil"),
    ("one_back", ("back",), "path"),
)

ENC_CFG = dict(hidden_size=32, num_hidden_layers=2, num_attention_heads=2, mlp_ratio=2, patch_size=14, image_size=56,
               use_swiglu_ffn=True, layerscale_value=1.0, qkv_bias=True, hidden_act="gelu", layer_norm_eps=1e-6)
ENC_IMAGE_SIZE = 56
ENC_SEED = 7
TABLE_WIDTHS = (1536, ENC_CFG["hidden_size"])

# (case name, B, V, view_idxs or None)
ENC_CASES = (
    ("b1_v1", 1, 1, None),
    ("b1_v1_idx", 1, 1, [(2,)]),
    ("b1_v2", 1, 2, None),
    ("b1_v2_idx", 1, 2, [(1, 3)]),
    ("b1_v4", 1, 4, None),
    ("b1_v4_idx", 1, 4, [(0, 1, 2, 3)]),
    ("b2_v1", 2, 1, None),
    ("b2_v1_idx", 2, 1, [(3,), (0,)]),
    ("b2_v2", 2, 2, None),
    ("b2_v2_idx", 2, 2, [(0, 2), (1, 3)]),
    ("b2_v4", 2, 4, None),
    ("b2_v4_idx", 2, 4, [(0, 1, 2, 3), (3, 2, 1, 0)]),
)


def sha(t):
    return np.array(hashlib.sha256(np.ascontiguousarray(np.asarray(t)).tobytes()).hexdigest())


def view_image(tag):
    """A seeded RGBA view: noise RGB inside an ellipse whose size and place differ per view (so a wrong view order
    changes the stacked tensor)."""
    from PIL import Image
    i = TAGS.index(tag)
    rng = np.random.default_rng(100 + i)
    h, w = 180 + 20 * i, 240 - 10 * i
    yy, xx = np.mgrid[0:h, 0:w]
    rgba = np.zeros((h, w, 4), np.uint8)
    rgba[..., :3] = rng.integers(0, 256, (h, w, 3))
    rgba[..., 3] = ((((xx - w * (0.4 + 0.05 * i)) / (w * 0.3)) ** 2 + ((yy - h * 0.5) / (h * (0.25 + 0.04 * i))) ** 2)
                    <= 1) * 255
    return Image.fromarray(rgba, "RGBA")


def proc_input(tags, kind, tmp):
    """The dict a PROC_CASES entry passes to the processor; path inputs are PNGs written under `tmp`."""
    out = {}
    for tag in tags:
        im = view_image(tag)
        if kind == "path":
            p = os.path.join(tmp, f"{tag}.png")
            im.save(p)
            im = p
        out[tag] = im
    return out


def enc_image(B, V):
    g = torch.Generator().manual_seed(1000 * B + V)
    return torch.rand(B, V, 3, 70, 90, generator=g) * 2 - 1


def enc_state_dict(keys, shapes, seed=ENC_SEED):
    """Seeded weights for the small encoder: N(0, 0.1) everywhere, norm weights and LayerScale gains near 1."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in zip(keys, shapes):
        v = torch.randn(tuple(shp), generator=g) * 0.1
        if k.endswith("lambda1") or ("norm" in k and k.endswith("weight")):
            v = v + 1.0
        sd[k] = v
    return sd


def load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def main():
    assert ref_import.available(), "reference checkout not found"
    z = {}
    proc = ref_import.hunyuan_preprocessors().MVImageProcessorV2(size=512, border_ratio=0.15)
    with tempfile.TemporaryDirectory() as tmp:
        for name, tags, kind in PROC_CASES:
            b = proc(proc_input(tags, kind, tmp))
            img, mask = b["image"].numpy(), b["mask"].numpy()
            z[f"proc_{name}_view_idxs"] = np.array(b["view_idxs"], np.int64)
            z[f"proc_{name}_image_shape"], z[f"proc_{name}_mask_shape"] = np.array(img.shape), np.array(mask.shape)
            z[f"proc_{name}_image_dtype"], z[f"proc_{name}_mask_dtype"] = np.array(str(img.dtype)), np.array(str(mask.dtype))
            z[f"proc_{name}_image_sha256"], z[f"proc_{name}_mask_sha256"] = sha(img), sha(mask)
    cref = load(os.path.join(ref_import.HY, "hy3dgen/shapegen/models/conditioner.py"), "_ref_conditioner")
    for C in TABLE_WIDTHS:
        cfg = dict(ENC_CFG, hidden_size=C, num_attention_heads=C // 16)
        t = cref.DinoImageEncoderMV(config=cfg, use_cls_token=True, image_size=ENC_IMAGE_SIZE, view_num=4)
        ve = t.view_embed                                   # [1, view_num, num_patches, C] float32
        assert ve.dtype == torch.float32 and all(torch.equal(ve[0, :, 0], ve[0, :, p]) for p in range(ve.shape[2]))
        z[f"table_{C}"] = ve[0, :, 0].numpy()
    torch.manual_seed(0)
    theirs = cref.DinoImageEncoderMV(config=ENC_CFG, use_cls_token=True, image_size=ENC_IMAGE_SIZE, view_num=4)
    sd0 = theirs.model.state_dict()
    keys = list(sd0)
    theirs.model.load_state_dict(enc_state_dict(keys, [tuple(v.shape) for v in sd0.values()]), strict=True)
    with torch.no_grad():
        for name, B, V, idxs in ENC_CASES:
            z[f"enc_{name}"] = theirs(enc_image(B, V), view_idxs=idxs).numpy()
        z["enc_uncond_b2_v3"] = theirs.unconditional_embedding(2, view_idxs=[(0, 1, 2), (0, 2, 3)]).numpy()
    np.savez_compressed(OUT, **z)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    torch.set_num_threads(8)
    main()
