"""GPU: the Hunyuan3D-2mini denoiser (HunYuanDiTPlain) on r3g -- the grouped expert GEMM (r3g_linear moe_mode; the
route and combine modes are checked in test_gpu_kernel_bounds.py), the whole DiT against the float32 oracle
(oracle/hy3d_mini_ref.py) on the routing the kernels chose, CUDA-graph replay, and image -> mesh with the 2mini
configuration."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

pytestmark = pytest.mark.gpu


def _ops():
    from r3g import ops
    return ops


GROUPED_COUNTS = {"uniform": [300, 300, 300, 300], "one_expert": [300, 0, 0, 0], "empty_expert": [129, 0, 257, 64],
                  "one_row": [1, 1, 0, 1], "ragged": [127, 131, 200, 5]}


@pytest.mark.parametrize("dist", list(GROUPED_COUNTS) + ["no_bias", "no_experts", "strided", "n8", "k200"])
def test_grouped_gemm_is_per_expert_linear_bit_for_bit(dist):
    """Each group equals ops.linear of its rows bit for bit, and the fp16_ref mirror, with and without the row scale.
    The cases past the row distributions take the ragged one and change one thing: no bias; experts = 0 (every group
    has cap rows); x and out strided views of wider buffers; N = 8 (one partial column tile); K = 200."""
    import fp16_ref as R
    ops = _ops()
    torch.manual_seed(1)
    G, cap = 5, 300
    E = 0 if dist == "no_experts" else 4
    N = 8 if dist == "n8" else 384
    K = 200 if dist == "k200" else 256
    counts = GROUPED_COUNTS.get(dist, GROUPED_COUNTS["ragged"])
    strided = dist == "strided"
    xbuf = torch.randn(G * cap, K + 40, device="cuda").half()
    x = xbuf[:, 16:16 + K] if strided else xbuf[:, :K].contiguous()
    w = (torch.randn(G, N, K, device="cuda") * 0.05).half()
    b = None if dist == "no_bias" else (torch.randn(G, N, device="cuda") * 0.1).half()
    scale = torch.rand(G * cap, device="cuda").half()
    cnt = torch.tensor(counts, device="cuda", dtype=torch.int32)
    # ops.linear takes N % 32 == 0: the reference pads w (and bias) with zero rows and keeps the first N columns
    Np = -(-N // 32) * 32
    wp = torch.zeros(G, Np, K, device="cuda", dtype=torch.float16)
    wp[:, :N] = w
    bp = None if b is None else torch.zeros(G, Np, device="cuda", dtype=torch.float16)
    if bp is not None:
        bp[:, :N] = b
    for act, rs in ((ops.ACT_GELU_ERF, None), (ops.ACT_NONE, scale)):
        obuf = torch.full((G * cap, N + 24), float("nan"), device="cuda", dtype=torch.float16)
        out = obuf[:, 8:8 + N] if strided else obuf[:, :N].contiguous()
        ops.moe_grouped(x, w, b, counts=cnt, experts=E, out=out, act=act, row_scale=rs)
        for g in range(G):
            n = counts[g] if g < E else cap
            if n == 0:
                continue
            rows = slice(g * cap, g * cap + n)
            bg = None if b is None else b[g]
            ref = ops.linear(x[rows], wp[g], None if bp is None else bp[g], act=act)[:, :N]
            if rs is not None:
                ref = ref * rs[rows, None]
            assert torch.equal(out[rows], ref), (dist, g, act)
            R.check_bound(out[rows], *R.linear(x[rows], w[g], bg, act=act, row_scale=None if rs is None else rs[rows]),
                          f"grouped {dist} group {g} act={act} scaled={rs is not None}")
        # rows past a group's count are not written, nor is anything outside the out view
        for g in range(E):
            assert torch.isnan(out[g * cap + counts[g]:(g + 1) * cap]).all()
        if strided:
            assert torch.isnan(obuf[:, :8]).all() and torch.isnan(obuf[:, 8 + N:]).all()


def test_moe_block_matches_the_oracle_on_the_kernel_routing():
    import hy3d_mini_ref as ref
    from r3g.dit_plain import HunYuanDiTPlain
    m = HunYuanDiTPlain(in_channels=64, hidden_size=256, context_dim=128, depth=2, num_heads=4, qk_norm=True,
                        use_attention_pooling=False, num_moe_layers=1, num_experts=4, moe_top_k=2).init_random(3)
    ws = m._workspace(2, 100, 40)
    M, H = 2 * 101, 256
    torch.manual_seed(2)
    h = torch.randn(M, 2 * H, device="cuda").half()
    s = h[:, H:]
    before = s.float().clone()
    m._moe(ws, "blocks.1.moe.", s, M)
    sd = {k_: v.float().cuda() for k_, v in m.reference_state_dict().items()}
    y = torch.nn.functional.layer_norm(before, (H,), sd["blocks.1.norm3.weight"], sd["blocks.1.norm3.bias"], 1e-6)
    want = before + ref.moe(sd, "blocks.1.moe.", y, ws["ids"].long(), ws["wts"], 4)
    err = (s.float() - want).abs().max().item()
    print(f"MoE block max |err| {err:.3e}, max |ref| {want.abs().max().item():.3f}")
    assert err < 2e-3 * want.abs().max().item()


def _model(depth, H=256, seed=0, **kw):
    from r3g.dit_plain import HunYuanDiTPlain
    cfg = dict(in_channels=64, hidden_size=H, context_dim=192, depth=depth, num_heads=H // 64, qk_norm=True,
               use_attention_pooling=False, qkv_bias=True, num_moe_layers=2, num_experts=4, moe_top_k=2)
    cfg.update(kw)
    return HunYuanDiTPlain(**cfg).init_random(seed), cfg


def _inputs(B, Li, Lt, C, cdim, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(B, Li, C, generator=g).half().cuda()
    cond = torch.randn(B, Lt, cdim, generator=g).half().cuda()
    t = torch.tensor([0.37, 0.81][:B], dtype=torch.float16).cuda()
    return x, t, cond


@pytest.mark.parametrize("depth", [5, 6])
def test_dit_matches_the_float32_oracle_per_block(depth):
    import hy3d_mini_ref as ref
    m, cfg = _model(depth, seed=depth)
    x, t, cond = _inputs(2, 200, 77, 64, 192)
    m.taps, m.routes = [], []
    out = m(x, t, {"main": cond})
    sd = {k: v.float().cuda() for k, v in m.reference_state_dict().items()}
    taps = []
    want = ref.forward(sd, cfg, x, t, cond, routes=[(i, w) for i, w in m.routes], taps=taps)
    for i, (a, b) in enumerate(zip(m.taps, taps)):
        rel = (a.float() - b).abs().max().item() / b.abs().max().item()
        print(f"depth {depth} block {i}: rel err {rel:.2e}")
        assert rel < 5e-3, (i, rel)
    rel = (out.float() - want).abs().max().item() / want.abs().max().item()
    print(f"depth {depth} output: rel err {rel:.2e}")
    assert rel < 5e-3


@pytest.mark.parametrize("depth", [2, 16])
def test_full_width_assumed_config_vs_oracle(depth):
    import hy3d_mini_ref as ref
    from r3g.pipelines import HUNYUAN3D_2MINI_CONFIG
    cfg = dict(HUNYUAN3D_2MINI_CONFIG["model"], depth=depth, num_moe_layers=min(6, depth - 1))
    cfg.pop("target")
    from r3g.dit_plain import HunYuanDiTPlain
    m = HunYuanDiTPlain(**cfg).init_random(7)
    x, t, cond = _inputs(2, 512, 1370, 64, 1024, seed=1)
    m.routes = []
    out = m(x, t, {"main": cond})
    sd = {k: v.float().cuda() for k, v in m.reference_state_dict().items()}
    want = ref.forward(sd, cfg, x, t, cond, routes=m.routes)
    rel = (out.float() - want).abs().max().item() / want.abs().max().item()
    print(f"full width depth {depth}: rel err {rel:.2e}")
    assert rel < 5e-3


def test_repeated_forwards_and_graph_replay_are_bit_identical():
    from r3g.graphs import GraphCache
    m, _ = _model(5)
    x, t, cond = _inputs(2, 200, 77, 64, 192)
    a = m(x, t, {"main": cond}).clone()
    b = m(x, t, {"main": cond}).clone()
    assert torch.equal(a, b)
    gc = GraphCache(keep_all=True)
    g = gc.get(("k",), (x, t, cond), lambda xs, ts, cs: m(xs, ts, {"main": cs}))
    g.inputs[0].copy_(x); g.inputs[1].copy_(t); g.inputs[2].copy_(cond)
    g.replay()
    assert torch.equal(g.outputs, a)
    g_first = g.outputs.clone()
    # a different context through the same graph matches a fresh eager forward
    x2, t2, cond2 = _inputs(2, 200, 77, 64, 192, seed=5)
    g.inputs[0].copy_(x2); g.inputs[1].copy_(t2); g.inputs[2].copy_(cond2)
    g.replay()
    replayed = g.outputs.clone()
    eager = m(x2, t2, {"main": cond2}).clone()
    assert torch.equal(replayed, eager) and not torch.equal(replayed, g_first)
    # the context's k / v projected once (project_context) and passed in gives the same bits
    kv = m.project_context(cond2)
    assert torch.equal(m(x2, t2, {"main": cond2}, context_kv=kv), eager)


def test_pipeline_image_to_mesh_with_the_2mini_config():
    sys.path.insert(0, ROOT)
    from bench import synthetic_crop
    from r3g.pipelines import HUNYUAN3D_2MINI_CONFIG, Hunyuan3DDiTFlowMatchingPipeline
    from r3g.dit_plain import HunYuanDiTPlain
    pipe = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=0, config=HUNYUAN3D_2MINI_CONFIG)
    assert isinstance(pipe.model, HunYuanDiTPlain)
    meshes = []
    for seed in (1, 2):
        out = pipe(image=synthetic_crop(seed), num_inference_steps=3, octree_resolution=64,
                   generator=torch.manual_seed(1234), output_type="mesh")[0]
        meshes.append(out)
    # the second call reuses the first call's graph with another image: it matches an eager call
    pipe.use_cuda_graph = False
    eager = pipe(image=synthetic_crop(2), num_inference_steps=3, octree_resolution=64,
                 generator=torch.manual_seed(1234), output_type="mesh")[0]
    for m in (meshes[1], eager):
        assert m is not None and len(m.mesh_f) > 0
    import numpy as np
    assert np.array_equal(np.asarray(meshes[1].mesh_v), np.asarray(eager.mesh_v))
    assert np.array_equal(np.asarray(meshes[1].mesh_f), np.asarray(eager.mesh_f))


def test_stage3_twin_runs_mini_random_weights(tmp_path):
    import subprocess
    import yaml
    sys.path.insert(0, ROOT)
    from bench import synthetic_crop
    inp, out = tmp_path / "in", tmp_path / "out"
    inp.mkdir()
    out.mkdir()
    synthetic_crop(1).save(inp / "chair__1.png")
    cfg = dict(use_banana=False, input_folder_hy=str(inp), output_folder_hy=str(out), num_inf_steps_hy=3,
               octree_resolution_hy=64, num_chunks_hy=16000, seed=1234567, mini=True)
    (tmp_path / "config.yaml").write_text(yaml.safe_dump(cfg))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "stages", "2d_to_3d_models", "run.py"), "--config",
                        str(tmp_path / "config.yaml"), "--random-weights"], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "wrote 1 mesh(es)" in r.stdout or "no surface" in r.stdout, r.stdout[-2000:]


def test_qk_rmsnorm_mode_is_torch_rmsnorm():
    """r3g_qk_norm mode 2 is nn.RMSNorm(64, eps=1e-6) on fp16 heads (HunYuanDiTPlain's q/k norms): one rounding of
    x * rrms * w.  It equals torch's fp16 module except where the two fp32 sums of squares, added in different orders,
    give rrms values one fp32 ulp apart and x * rrms * w sits on an fp16 rounding boundary: at most 1 in 10 000 elements,
    each by a rounding step.  Mode 0 (the 2.0 DiT's QKNorm, rounded before the scale) differs on a large share."""
    ops = _ops()
    torch.manual_seed(3)
    nh = 4
    buf = (torch.randn(3000, 3 * nh * 64, device="cuda") * 3).half()
    qw, kw = (1 + 0.3 * torch.randn(64, device="cuda")).half(), (1 + 0.3 * torch.randn(64, device="cuda")).half()
    norm_q = torch.nn.RMSNorm(64, eps=1e-6, device="cuda", dtype=torch.float16)
    norm_k = torch.nn.RMSNorm(64, eps=1e-6, device="cuda", dtype=torch.float16)
    with torch.no_grad():
        norm_q.weight.copy_(qw)
        norm_k.weight.copy_(kw)
        want_q = norm_q(buf[:, :nh * 64].view(-1, nh, 64)).view(-1, nh * 64)
        want_k = norm_k(buf[:, nh * 64:2 * nh * 64].view(-1, nh, 64)).view(-1, nh * 64)
    out = buf.clone()
    ops.qk_norm_(out, nh, 0, nh * 64, 64, 2, 1e-6, qw, None, kw, None)
    bad = (out[:, :nh * 64] != want_q).sum().item() + (out[:, nh * 64:2 * nh * 64] != want_k).sum().item()
    print(f"nn.RMSNorm mode: {bad} of {2 * want_q.numel()} elements differ")
    assert bad <= 2 * want_q.numel() // 10000
    for got, want in ((out[:, :nh * 64], want_q), (out[:, nh * 64:2 * nh * 64], want_k)):
        d = (got.double() - want.double()).abs()
        print(f"largest difference {d.max().item():.3e} at |value| {want.double().abs().flatten()[d.argmax()].item():.3e}")
        assert (d <= 2e-3 * want.double().abs().clamp_min(1e-2)).all()
    assert torch.equal(out[:, 2 * nh * 64:], buf[:, 2 * nh * 64:])
    old = buf.clone()
    ops.qk_norm_(old, nh, 0, nh * 64, 64, 0, 1e-6, qw, None, kw, None)
    old_bad = (old[:, :nh * 64] != want_q).sum().item()
    print(f"QKNorm mode: {old_bad} of {want_q.numel()} q elements differ")
    assert old_bad > 100 * bad + 1000


@pytest.mark.parametrize("name", ["odd", "even"])
def test_dit_matches_the_reference_fixture_per_block(name):
    """The DiT on the weights and inputs of tests/golden/hunyuandit_plain_mini.npz (the reference's own HunYuanDiTPlain
    and MoEBlock in float32): the same experts for every row, and every block's hidden state and the output within
    fp16 tolerance."""
    import numpy as np
    import hy3d_mini_ref as R
    from r3g.dit_plain import HunYuanDiTPlain
    z = np.load(os.path.join(ROOT, "tests", "golden", "hunyuandit_plain_mini.npz"))
    sd = R.mini_state_dict(z[f"{name}_w_keys"], z[f"{name}_w_shapes"], int(z[f"{name}_w_seed"]))
    m = HunYuanDiTPlain(in_channels=64, hidden_size=128, context_dim=96, depth=int(z[f"{name}_depth"]), num_heads=2,
                        qk_norm=True, qk_norm_type="rms", use_attention_pooling=False,
                        qkv_bias=bool(z[f"{name}_qkv_bias"]), num_moe_layers=2, num_experts=4, moe_top_k=2)
    m.load_state_dict(sd)
    x, t, cond = (torch.from_numpy(z[f"{name}_{k}"]).cuda() for k in ("x", "t", "cond"))
    m.taps, m.routes = [], []
    out = m(x, t, {"main": cond})
    for i, (ids, w) in enumerate(m.routes):
        ref_ids = torch.from_numpy(z[f"{name}_gate{i}_ids"]).long().cuda()
        assert torch.equal(ids.long().sort(-1).values, ref_ids.sort(-1).values), (name, i)
        ref_w = torch.from_numpy(z[f"{name}_gate{i}_w"]).cuda()
        assert (w.float().sort(-1).values - ref_w.sort(-1).values).abs().max() < 5e-3
    for i, tp in enumerate(m.taps):
        ref = torch.from_numpy(z[f"{name}_tap{i}"]).cuda()
        rel = ((tp.float() - ref).abs().max() / ref.abs().max()).item()
        print(f"{name} block {i}: rel err {rel:.2e}")
        assert rel < 5e-3, (name, i, rel)
    ref = torch.from_numpy(z[f"{name}_y"]).cuda()
    rel = ((out.float() - ref).abs().max() / ref.abs().max()).item()
    print(f"{name} output: rel err {rel:.2e}")
    assert rel < 5e-3
