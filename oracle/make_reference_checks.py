"""ORACLE -- fixture generator (needs the reference checkout, see oracle/ref_import.py).

Runs the reference's own modules on the inputs of the host-side comparison tests and stores what those tests compare
against in tests/golden/reference_checks.npz, so that the tests run anywhere:
  imgproc_*   ImageProcessorV2 (preprocessors.py) on a seeded RGBA image: sha256 of the image / mask + a seeded sample
  cond_*      DinoImageEncoder (conditioner.py:57-131): a small random model's weights, its outputs on seeded inputs
  nsm_*       extract_near_surface_volume_fn (volume_decoders.py:29-119) on seeded volumes
  helper_*    vggt/utils/helper.py: create_pixel_coordinate_grid, randomly_limit_trues
  loader_*    load_and_preprocess_images_square (vggt/utils/load_fn.py:13-94) on seeded PNGs: sha256 + sample, coords
  ckpt_*      state-dict keys and shapes of the reference's Hunyuan3DDiT / Transformer / CrossAttentionDecoder
  heads_*     CameraHead / DPTHead / pose_encoding_to_extri_intri on seeded weights (per-tensor mean / std of the
              reference's initialisation, redrawn from a seeded generator) and seeded tokens

  python oracle/make_reference_checks.py
"""
import hashlib
import importlib.util
import os
import sys
import tempfile
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import ref_import  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference_checks.npz")


def sha(t):
    return np.array(hashlib.sha256(np.ascontiguousarray(np.asarray(t)).tobytes()).hexdigest())


def sample_idx(n, k=4096):
    return np.sort(np.random.default_rng(0).choice(n, size=min(k, n), replace=False))


def load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


# ---- inputs shared with the tests (tests/test_host_logic.py, tests/test_stage4_tail.py, ...)
def imgproc_input():
    from PIL import Image
    rng = np.random.default_rng(0)
    rgba = np.zeros((300, 420, 4), np.uint8)
    rgba[..., :3] = rng.integers(0, 256, (300, 420, 3))
    yy, xx = np.mgrid[0:300, 0:420]
    rgba[..., 3] = ((((xx - 200) / 120) ** 2 + ((yy - 160) / 90) ** 2) <= 1) * 255
    return Image.fromarray(rgba, "RGBA")


COND_CFG = dict(hidden_size=32, num_hidden_layers=2, num_attention_heads=2, mlp_ratio=2, patch_size=14, image_size=56,
                use_swiglu_ffn=True, layerscale_value=1.0, qkv_bias=True, hidden_act="gelu", layer_norm_eps=1e-6)
COND_SHAPES = ((1, 3, 70, 90), (2, 3, 100, 64), (1, 3, 56, 56))


def cond_inputs():
    g = torch.Generator().manual_seed(0)
    return [torch.rand(s, generator=g) * 2 - 1 for s in COND_SHAPES]


def nsm_inputs():
    g = torch.Generator().manual_seed(0)
    out = {}
    for n in (5, 9):
        x = torch.randn(n, n, n, generator=g)
        x[torch.rand(n, n, n, generator=g) < 0.25] = -10000.0
        out[n] = x
    return out


NSM_ALPHAS = (0.0, 0.3, -0.2)


def loader_images(tmp):
    from PIL import Image
    rng = np.random.default_rng(9)
    paths = []
    for i, (w, h, mode) in enumerate(((150, 100, "RGB"), (64, 97, "RGBA"), (80, 80, "RGB"))):
        arr = rng.integers(0, 256, (h, w, 4 if mode == "RGBA" else 3)).astype(np.uint8)
        pth = os.path.join(tmp, f"im{i}.png")
        Image.fromarray(arr, mode).save(pth)
        paths.append(pth)
    return paths


HEADS_C, HEADS_S, HEADS_H, HEADS_W = 128, 2, 56, 70


def heads_inputs():
    g = torch.Generator().manual_seed(1)
    ph, pw = HEADS_H // 14, HEADS_W // 14
    toks = [torch.randn(1, HEADS_S, 5 + ph * pw, HEADS_C, generator=g) for _ in range(4)]
    imgs = torch.rand(1, HEADS_S, 3, HEADS_H, HEADS_W, generator=g)
    return toks, imgs


def redraw(stats_keys, stats, shapes, seed):
    """state dict from per-tensor (mean, std): a seeded normal draw, in key order."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, (m, s), shp in zip(stats_keys, stats, shapes):
        sd[str(k)] = torch.randn(shape_of(shp), generator=g) * float(s) + float(m)
    return sd


def stats_of(sd):
    keys, st, shapes = [], [], []
    for k, v in sd.items():
        v = v.float()
        keys.append(k)
        st.append((v.mean().item(), v.std().item() if v.numel() > 1 else 0.0))
        shapes.append(list(v.shape) + [0] * (4 - v.dim()))
    return np.array(keys), np.array(st, np.float64), np.array(shapes, np.int64)


def shape_of(row):
    return tuple(int(x) for x in row if x > 0)


def main():
    assert ref_import.available(), "reference checkout not found"
    z = {}
    # ImageProcessorV2
    ref = ref_import.hunyuan_preprocessors().ImageProcessorV2(size=512, border_ratio=0.15)
    b = ref(imgproc_input())
    img, mask = b["image"].numpy(), b["mask"].numpy()
    z["imgproc_image_sha256"], z["imgproc_mask_sha256"] = sha(img), sha(mask)
    z["imgproc_image_shape"], z["imgproc_mask_shape"] = np.array(img.shape), np.array(mask.shape)
    z["imgproc_image_sample"] = img.reshape(-1)[sample_idx(img.size)]
    z["imgproc_image_dtype"], z["imgproc_mask_dtype"] = np.array(str(img.dtype)), np.array(str(mask.dtype))
    # DinoImageEncoder
    cref = load(os.path.join(ref_import.HY, "hy3dgen/shapegen/models/conditioner.py"), "_ref_conditioner")
    torch.manual_seed(0)
    theirs = cref.DinoImageEncoder(config=COND_CFG, use_cls_token=True, image_size=56)
    for k, v in theirs.model.state_dict().items():
        z["cond_w:" + k] = v.numpy()
    for i, x in enumerate(cond_inputs()):
        z[f"cond_out{i}"] = theirs(x).detach().numpy()
    z["cond_uncond"] = theirs.unconditional_embedding(2).numpy()
    # near-surface volume
    _, _, vd = ref_import.hunyuan_autoencoders()
    for n, x in nsm_inputs().items():
        for j, alpha in enumerate(NSM_ALPHAS):
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                z[f"nsm_{n}_{j}"] = vd.extract_near_surface_volume_fn(x.clone(), alpha).numpy()
    # VGGT helpers
    helper = load(os.path.join(ref_import.VGGT, "vggt/utils/helper.py"), "_ref_vggt_helper")
    z["helper_grid"] = helper.create_pixel_coordinate_grid(2, 5, 4)
    m = np.random.default_rng(3).random((2, 30, 30)) > 0.3
    np.random.seed(7)
    z["helper_limit_trues"] = helper.randomly_limit_trues(m.copy(), 100)
    # image loader
    lf = load(os.path.join(ref_import.VGGT, "vggt/utils/load_fn.py"), "_ref_load_fn")
    with tempfile.TemporaryDirectory() as tmp:
        paths = loader_images(tmp)
        for tag, sel in (("all", paths), ("one", paths[:1])):
            a_img, a_xy = lf.load_and_preprocess_images_square(sel, 256)
            a_img = a_img.numpy()
            z[f"loader_{tag}_sha256"], z[f"loader_{tag}_shape"] = sha(a_img), np.array(a_img.shape)
            z[f"loader_{tag}_sample"] = a_img.reshape(-1)[sample_idx(a_img.size)]
            z[f"loader_{tag}_xy"] = a_xy.numpy()
    # checkpoint layout: key names and shapes of the reference's modules
    ref_dit = ref_import.hunyuan_dit()
    ab, _, _ = ref_import.hunyuan_autoencoders()
    dit = ref_dit.Hunyuan3DDiT(in_channels=64, context_in_dim=96, hidden_size=128, mlp_ratio=4.0, num_heads=2, depth=2,
                               depth_single_blocks=3, axes_dim=[64], theta=10000, qkv_bias=True, time_factor=1000,
                               guidance_embed=False)
    tr = ab.Transformer(n_ctx=48, width=128, layers=2, heads=2, qkv_bias=False, qk_norm=True)
    geo = ab.CrossAttentionDecoder(out_channels=1, num_latents=48, mlp_expand_ratio=4, downsample_ratio=1,
                                   enable_ln_post=True, fourier_embedder=ab.FourierEmbedder(num_freqs=8, include_pi=False),
                                   width=128, heads=2, qkv_bias=False, qk_norm=True, label_type="binary")
    for name, mod in (("dit", dit), ("tr", tr), ("geo", geo)):
        sd = mod.state_dict()
        z[f"ckpt_{name}_keys"] = np.array(list(sd.keys()))
        z[f"ckpt_{name}_shapes"] = np.array([list(v.shape) + [0] * (4 - v.dim()) for v in sd.values()], np.int64)
    # VGGT heads
    ref_import.vggt_package()
    from vggt.heads.camera_head import CameraHead as RefCam
    from vggt.heads.dpt_head import DPTHead as RefDPT
    from vggt.utils.pose_enc import pose_encoding_to_extri_intri as ref_pose
    torch.manual_seed(0)
    toks, imgs = heads_inputs()
    cam = RefCam(dim_in=HEADS_C, trunk_depth=2, num_heads=2).eval()
    with torch.no_grad():
        for n, p in cam.named_parameters():
            if "gamma" in n or n == "empty_pose_tokens":
                p.copy_(0.3 * torch.randn_like(p))
    keys, st, shapes = stats_of(cam.state_dict())
    z["heads_cam_keys"], z["heads_cam_stats"], z["heads_cam_shapes"] = keys, st, shapes
    cam.load_state_dict(redraw(keys, st, shapes, 2))
    dpt = RefDPT(dim_in=HEADS_C, output_dim=2, activation="exp", conf_activation="expp1", features=32,
                 out_channels=[16, 32, 64, 64], intermediate_layer_idx=[0, 1, 2, 3]).eval()
    keys, st, shapes = stats_of(dpt.state_dict())
    z["heads_dpt_keys"], z["heads_dpt_stats"], z["heads_dpt_shapes"] = keys, st, shapes
    dpt.load_state_dict(redraw(keys, st, shapes, 3))
    with torch.no_grad():
        cams = cam(toks)
        for i, c in enumerate(cams):
            z[f"heads_cam_out{i}"] = c.numpy()
        e, k = ref_pose(cams[-1], (HEADS_H, HEADS_W))
        z["heads_extri"], z["heads_intri"] = e.numpy(), k.numpy()
        d, c = dpt(toks, images=imgs, patch_start_idx=5)
        z["heads_depth"], z["heads_conf"] = d.numpy(), c.numpy()
    np.savez_compressed(OUT, **z)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
