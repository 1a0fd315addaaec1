"""GPU: the VGGT aggregator mirror (fp16 tensor-core operands, fp32 residual stream) against the fixture produced
by the reference's own Aggregator / DinoVisionTransformer modules, and at full width against the fp32 oracle.
Tolerance: the reference itself runs this under bf16 autocast (8 mantissa bits); we require rel-L2 <= 5e-3
against the fp32 ground truth."""
import gc
import os
import weakref

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.float().flatten().cpu(), b.float().flatten().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def test_qk_norm_rope_kernel_against_oracle():
    import vggt_ref as V
    from r3g import ops
    torch.manual_seed(0)
    Bf, hp, wp, H = 3, 4, 5, 2
    P = hp * wp + 5
    qkv = torch.randn(Bf * P, 3 * H * 64, device="cuda").half()
    qw, qb = (1 + 0.2 * torch.randn(64, device="cuda")).half(), (0.1 * torch.randn(64, device="cuda")).half()
    kw, kb = (1 + 0.2 * torch.randn(64, device="cuda")).half(), (0.1 * torch.randn(64, device="cuda")).half()
    ref = qkv.float().view(Bf, P, 3, H, 64).permute(2, 0, 3, 1, 4).clone()
    q = torch.nn.functional.layer_norm(ref[0], (64,), qw.float(), qb.float(), 1e-5)
    k = torch.nn.functional.layer_norm(ref[1], (64,), kw.float(), kb.float(), 1e-5)
    ys, xs = torch.meshgrid(torch.arange(hp), torch.arange(wp), indexing="ij")
    pos = torch.cat([torch.zeros(5, 2, dtype=torch.long), torch.stack((ys, xs), -1).reshape(-1, 2) + 1])[None].expand(Bf, -1, -1).cuda()
    q, k = V.rope_2d(q, pos, 100.0), V.rope_2d(k, pos, 100.0)
    out = ops.qk_norm_rope_(qkv.clone(), H, 1e-5, qw, qb, kw, kb, 100.0, P, 5, wp).float().view(Bf, P, 3, H, 64)
    assert (out[:, :, 0].permute(0, 2, 1, 3) - q).abs().max().item() < 6e-3
    assert (out[:, :, 1].permute(0, 2, 1, 3) - k).abs().max().item() < 6e-3
    assert torch.equal(out[:, :, 2], qkv.float().view(Bf, P, 3, H, 64)[:, :, 2])


def test_aggregator_and_dino_mini_against_reference_fixture(golden_dir):
    from r3g.vggt import Aggregator, DinoVisionTransformer
    z = np.load(os.path.join(golden_dir, "vggt_mini.npz"))
    sd = {k[len("w:agg."):]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w:agg.")}
    agg = Aggregator(img_size=56, patch_size=14, embed_dim=128, depth=2, num_heads=2, patch_embed="conv")
    agg.load_state_dict(sd)
    images = torch.from_numpy(z["agg_images"]).cuda()
    outs, psi = agg(images)
    assert psi == int(z["agg_psi"]) and len(outs) == 2
    for i, o in enumerate(outs):
        assert o.dtype == torch.float32 and tuple(o.shape) == z[f"agg_out{i}"].shape
        assert rel_l2(o, torch.from_numpy(z[f"agg_out{i}"])) < 5e-3
    # graph replay == eager launches; the graph keeps its workspace when an eager call of another shape replaces it
    graph_outs = [o.clone() for o in outs]
    captured = [weakref.ref(t) for t in next(iter(agg._ws.values())).values()]
    agg.use_cuda_graph = False
    eager, _ = agg(images)
    assert all(torch.equal(a, b) for a, b in zip(eager, graph_outs)), "graph replay must equal the eager launches"
    agg(images[:, :1])
    gc.collect()
    assert all(r() is not None for r in captured), "the graph must keep its captured workspace alive"
    agg.use_cuda_graph = True
    again, _ = agg(images)
    assert all(torch.equal(a, b) for a, b in zip(again, graph_outs))
    vsd = {k[len("w:vit."):]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w:vit.")}
    vit = DinoVisionTransformer(vsd, "", 128, 2, 2, 14, 4, torch.device("cuda"))
    for tag in ("native", "interp"):
        x = torch.from_numpy(z[f"vit_x_{tag}"]).cuda()
        n, _, hh, ww = x.shape
        rows = n * ((hh // 14) * (ww // 14) + 5)
        e = lambda *s: torch.empty(*s, device="cuda", dtype=torch.float16)  # noqa: E731
        ws = dict(xn=e(rows, 128), qkv=e(rows, 384), hid=e(rows, 512))
        y = vit.forward_patch_tokens(x, None, None, ws)
        assert rel_l2(y, torch.from_numpy(z[f"vit_y_{tag}"])) < 5e-3


def test_aggregator_full_width_against_oracle():
    """embed 1024 / 16 heads / 518x518 (1374 tokens per frame), S = 2, 2+2 alternating blocks, conv patch embed."""
    import vggt_ref as V
    from r3g.vggt import Aggregator
    torch.manual_seed(1)
    C, depth = 1024, 2
    sd = {"patch_embed.proj.weight": torch.randn(C, 3, 14, 14) * 0.02, "patch_embed.proj.bias": torch.randn(C) * 0.02,
          "camera_token": torch.randn(1, 2, 1, C) * 0.5, "register_token": torch.randn(1, 2, 4, C) * 0.5}
    for kind in ("frame", "global"):
        for i in range(depth):
            p = f"{kind}_blocks.{i}."
            for n, shp, s in (("attn.qkv", (3 * C, C), 0.02), ("attn.proj", (C, C), 0.02), ("mlp.fc1", (4 * C, C), 0.02),
                              ("mlp.fc2", (C, 4 * C), 0.02)):
                sd[p + n + ".weight"], sd[p + n + ".bias"] = torch.randn(*shp) * s, torch.randn(shp[0]) * 0.02
            for n, d in (("norm1", C), ("norm2", C), ("attn.q_norm", 64), ("attn.k_norm", 64)):
                sd[p + n + ".weight"], sd[p + n + ".bias"] = 1 + 0.1 * torch.randn(d), 0.05 * torch.randn(d)
            sd[p + "ls1.gamma"], sd[p + "ls2.gamma"] = 0.5 + 0.1 * torch.randn(C), 0.5 + 0.1 * torch.randn(C)
    sd = {k: v.half().float() for k, v in sd.items()}
    imgs = torch.rand(1, 2, 3, 518, 518, device="cuda")
    agg = Aggregator(depth=depth, patch_embed="conv").load_state_dict(sd)
    outs, _ = agg(imgs)
    ref = V.aggregator({k: v.cuda() for k, v in sd.items()}, imgs, depth, 16)
    for o, r in zip(outs, ref):
        assert rel_l2(o, r) < 5e-3


def test_run_vggt_composite_against_cpu_oracle():
    """row v2: aggregator (r3g kernels) -> camera head -> pose_encoding_to_extri_intri -> DPT depth head ->
    r3g_unproject, strung together by the stage twin's run_VGGT, against the fp32 CPU path: oracle aggregator, the same
    head mirrors on the CPU (pinned against the reference modules in tests/test_oracle_golden.py) and the oracle's
    numpy back-projection."""
    import importlib.util
    import hy3d_ref as R
    import vggt_ref as V
    from r3g import ops
    from r3g.vggt_heads import CameraHead, DPTHead, VGGT, pose_encoding_to_extri_intri, random_state_dict
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("stage4", os.path.join(root, "stages", "camera_and_pointcloud",
                                                                          "minimal_demo_vggt.py"))
    stage4 = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(stage4)
    C, depth = 128, 2
    sd = random_state_dict(3, embed_dim=C, depth=depth, vit_depth=2, trunk_depth=2, features=32,
                           out_channels=(32, 64, 128, 128), img_size=56)
    sd = {k: v.half().float() for k, v in sd.items()}
    hk, dk = dict(trunk_depth=2, num_heads=4), dict(intermediate_layer_idx=(0, 1, 0, 1))
    model = VGGT(img_size=56, embed_dim=C, depth=depth, num_heads=2, vit_depth=2, patch_embed="dinov2_vits14_reg",
                 camera_head_kwargs=hk, depth_head_kwargs=dk).load_state_dict(sd)
    torch.manual_seed(0)
    images = torch.rand(2, 3, 112, 112)
    E, K, dmap, conf = stage4.run_VGGT(model, images.cuda(), resolution=56)
    pts = ops.unproject(dmap[..., 0].contiguous(), E, K, torch.float64).cpu().numpy()
    # CPU fp32 path
    im = torch.nn.functional.interpolate(images, size=(56, 56), mode="bilinear", align_corners=False)[None]
    asd = {k[len("aggregator."):]: v for k, v in sd.items() if k.startswith("aggregator.")}
    toks = V.aggregator(asd, im, depth, 2, vit_depth=2)
    pose = CameraHead(sd, device="cpu", **hk)(toks)[-1]
    Er, Kr = pose_encoding_to_extri_intri(pose, im.shape[-2:])
    dr, cr = DPTHead(sd, device="cpu", **dk)(toks, im, 5)
    assert np.abs(E - Er[0].numpy()).max() < 5e-3 and np.abs(K - Kr[0].numpy()).max() < 5e-2 * np.abs(Kr[0].numpy()).max()
    assert rel_l2(dmap, dr[0]) < 1e-2 and rel_l2(conf, cr[0]) < 1e-2
    ref_pts = R.unproject_depth_map_to_point_map(dmap.cpu().numpy(), E, K)
    assert pts.dtype == np.float64 and np.array_equal(pts, ref_pts)      # the back-projection itself is exact


def test_camera_head_on_r3g_kernels_against_the_torch_mirror():
    """row v4: CameraHeadR3G (fp16 weights, float32 activations, GEMV / LayerNorm / small-attention kernels, one CUDA graph)
    vs the float32 torch mirror that tests/test_oracle_golden.py pins against the reference module -- full geometry
    (2048 wide, 16 heads of 128, 4 trunk blocks, 4 iterations) and a small one; graph replay == eager."""
    from r3g import ops
    from r3g.vggt_heads import CameraHead, CameraHeadR3G, random_state_dict
    # the three kernels alone
    torch.manual_seed(0)
    w = (torch.randn(96, 64, device="cuda") * 0.1)
    b, x, res, gm = (torch.randn(*s, device="cuda") for s in ((96,), (3, 64), (3, 96), (96,)))
    got = ops.gemv_f32(w.half(), b, x, residual=res, gamma=gm, silu_in=True, gelu_out=True)
    ref = res + gm * torch.nn.functional.gelu(torch.nn.functional.silu(x) @ w.half().float().t() + b)
    assert (got - ref).abs().max().item() < 1e-4
    xs = torch.randn(5, 200, device="cuda")
    lw, lb, sh, sc, gt = (torch.randn(*s, device="cuda") for s in ((200,), (200,), (5, 200), (5, 200), (5, 200)))
    ln = torch.nn.functional.layer_norm
    assert (ops.layernorm_f32(xs, lw, lb, eps=1e-5) - ln(xs, (200,), lw, lb, 1e-5)).abs().max().item() < 1e-4
    assert (ops.layernorm_f32(xs, eps=1e-6, shift=sh, scale=sc, gate=gt)
            - (gt * (ln(xs, (200,), eps=1e-6) * (1 + sc) + sh) + xs)).abs().max().item() < 1e-4
    qkv = torch.randn(2 * 5, 3 * 4 * 128, device="cuda")
    q, k, v = qkv.view(2, 5, 3, 4, 128).permute(2, 0, 3, 1, 4)
    ref = torch.nn.functional.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(10, 512)
    assert (ops.small_attention_f32(qkv, 2, 5, 4, 128) - ref).abs().max().item() < 1e-4
    # the whole head
    for C, heads, trunk in ((1024, 16, 4), (128, 2, 2)):
        sd = random_state_dict(7, embed_dim=C, depth=1, vit_depth=1, trunk_depth=trunk, features=32,
                               out_channels=(32, 64, 128, 128), img_size=56)
        sd = {k: v for k, v in sd.items() if k.startswith("camera_head.")}
        mine = CameraHeadR3G(sd, trunk_depth=trunk, num_heads=heads)
        mirror = CameraHead({k: (v.half().float() if v.dim() == 2 and v.shape[1] % 8 == 0 else v) for k, v in sd.items()},
                            trunk_depth=trunk, num_heads=heads, device="cuda")
        toks = [torch.randn(1, 2, 7, 2 * C, device="cuda")]
        a = mine(toks)
        b_ = mirror(toks)
        mine.use_cuda_graph = False
        c = mine(toks)
        for x1, x2, x3 in zip(a, b_, c):
            assert torch.equal(x1, x3), "graph replay must equal the eager launches"
            assert (x1 - x2).abs().max().item() < 2e-3 * max(1.0, x2.abs().max().item())


def test_conv_kernels_against_torch():
    """im2col3x3 + linear == F.conv2d (stride 1 and 2, ReLU epilogue, residual), bilinear_nhwc == F.interpolate
    (align_corners=True), on channels-last fp16."""
    import torch.nn.functional as F
    from r3g import ops
    torch.manual_seed(0)
    N, H, W, C, Co = 2, 13, 17, 64, 96
    x = torch.randn(N, H, W, C, device="cuda").half()
    wt = (torch.randn(Co, C, 3, 3, device="cuda") * 0.05).half()
    b = (torch.randn(Co, device="cuda") * 0.1).half()
    wm = wt.permute(0, 2, 3, 1).reshape(Co, 9 * C).contiguous()
    for stride in (1, 2):
        cols, Ho, Wo = ops.im2col3x3(x, stride=stride)
        y = ops.linear(cols, wm, b, act=ops.ACT_RELU).view(N, Ho, Wo, Co)
        ref = F.relu(F.conv2d(x.permute(0, 3, 1, 2).float(), wt.float(), b.float(), stride=stride, padding=1)).permute(0, 2, 3, 1)
        assert y.shape == ref.shape and (y.float() - ref).abs().max().item() < 2e-2 * ref.abs().max().item()
    cols, Ho, Wo = ops.im2col3x3(x, relu_in=True)
    res = torch.randn(N * H * W, Co, device="cuda").half()
    y = ops.linear(cols, wm, b, residual=res)
    ref = F.conv2d(F.relu(x.permute(0, 3, 1, 2).float()), wt.float(), b.float(), padding=1).permute(0, 2, 3, 1).reshape(-1, Co) + res.float()
    assert (y.float() - ref).abs().max().item() < 2e-2 * ref.abs().max().item()
    for size in ((26, 34), (19, 23), (13, 17)):
        got = ops.bilinear_nhwc(x, *size)
        ref = F.interpolate(x.permute(0, 3, 1, 2).float(), size=size, mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
        assert (got.float() - ref).abs().max().item() < 4e-3


def test_dpt_head_on_r3g_kernels_against_the_torch_mirror():
    """row v6: DPTHeadR3G (every convolution a wgmma GEMM over NHWC fp16) vs the float32 torch mirror that
    tests/test_oracle_golden.py pins against the reference module; the real channel widths at a 70 x 84 image, and a
    small one.  Graph replay == eager."""
    from r3g.vggt_heads import DPTHead, DPTHeadR3G, random_state_dict
    for C, feats, ocs, hw in ((1024, 256, (256, 512, 1024, 1024), (70, 84)), (128, 32, (32, 64, 128, 128), (56, 56))):
        sd = random_state_dict(5, embed_dim=C, depth=1, vit_depth=1, trunk_depth=1, features=feats, out_channels=ocs, img_size=56)
        sd = {k: v.half().float() for k, v in sd.items() if k.startswith("depth_head.")}
        H, W = hw
        P = (H // 14) * (W // 14)
        torch.manual_seed(1)
        toks = [torch.randn(1, 2, 5 + P, 2 * C, device="cuda") for _ in range(2)]
        imgs = torch.rand(1, 2, 3, H, W, device="cuda")
        kw = dict(intermediate_layer_idx=(0, 1, 0, 1))
        mine, mirror = DPTHeadR3G(sd, **kw), DPTHead(sd, device="cuda", **kw)
        d1, c1 = mine(toks, imgs, 5)
        d2, c2 = mirror(toks, imgs, 5)
        mine.use_cuda_graph = False
        d3, c3 = mine(toks, imgs, 5)
        assert d1.shape == d2.shape == (1, 2, H, W, 1) and c1.shape == c2.shape == (1, 2, H, W)
        assert torch.equal(d1, d3) and torch.equal(c1, c3), "graph replay must equal the eager launches"
        e_d, e_c = rel_l2(d1, d2), rel_l2(c1, c2)
        print(f"DPT on r3g kernels, width {C}: depth rel-L2 {e_d:.2e}, confidence rel-L2 {e_c:.2e}")
        assert e_d < 1e-2 and e_c < 1e-2
