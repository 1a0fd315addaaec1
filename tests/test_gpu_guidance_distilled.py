"""GPU: the guidance-distilled Hunyuan3D-2 path (`hunyuan3d-dit-v2-0-fast` / `-turbo`) on the r3g kernels -- the gemv
residual and the single-sample Euler step bit for bit, the guidance embedding and the guided DiT against fixtures from
the reference's own modules, the full model against the fp32 oracle, and the distilled pipeline end to end.

Tolerances are those of tests/test_gpu_models.py (mini DiT: per-block rel-L2 <= 3e-3, output <= 1e-2) and
tests/test_gpu_full_config.py (48 blocks: per-block <= 1e-2; latents after a few steps <= 3e-2)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MINI = dict(in_channels=64, context_in_dim=96, hidden_size=128, num_heads=2, depth=2, depth_single_blocks=2)


def rel_l2(a, b):
    a, b = a.float().flatten(), b.float().flatten()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def test_gemv_residual_bit_exact_and_may_alias_out():
    from r3g import ops
    torch.manual_seed(7)
    for B, silu_out in ((1, False), (2, True), (5, False)):
        w = (torch.randn(1024, 256, device="cuda") * 0.05).half()
        b = (torch.randn(1024, device="cuda") * 0.1).half()
        v = torch.randn(B, 256, device="cuda").half()
        res = torch.randn(B, 1024, device="cuda").half()
        plain = ops.gemv(w, b, v, silu_out=silu_out)
        # `vec + guidance_in(...)`: the fp16 GEMV result plus the fp16 residual, as torch adds two fp16 tensors
        want = plain + res
        got = ops.gemv(w, b, v, silu_out=silu_out, residual=res)
        assert torch.equal(got, want)
        inplace = res.clone()
        assert ops.gemv(w, b, v, silu_out=silu_out, residual=inplace, out=inplace) is inplace
        assert torch.equal(inplace, want)
        # residual=None is the plain GEMV
        assert torch.equal(ops.gemv(w, b, v, silu_out=silu_out, residual=None), plain)
    with pytest.raises(ValueError, match="residual"):
        ops.gemv(w, b, v, residual=res[:, :512])


def test_euler_step_without_cfg_bit_exact():
    import hy3d_ref as R
    from r3g import ops
    torch.manual_seed(3)
    x = torch.randn(1, 3072, 64).half()
    v = torch.randn(1, 3072, 64).half()
    for sig0, sig1 in ((0.5996, 0.7998), (0.7998, 1.0), (0.0, 0.0204)):
        s0, s1 = torch.tensor(sig0, dtype=torch.float32), torch.tensor(sig1, dtype=torch.float32)
        ref = R.flow_euler_step(x, v, s0, s1)           # schedulers.py:300-309 / :460-466, CPU dtype flow
        xd = x.cuda().clone()
        dup = torch.full((2, 3072, 64), 7.0, device="cuda", dtype=torch.float16)
        ops.cfg_euler_step_(xd, v.cuda(), 123.0, float((s1 - s0).half()), x_dup=dup[:1])   # guidance is ignored
        assert torch.equal(xd.cpu(), ref)
        assert torch.equal(dup[0], xd[0]) and (dup[1] == 7.0).all(), "x_dup must be written exactly once"
    with pytest.raises(ValueError, match="x_dup"):
        ops.cfg_euler_step_(x.cuda(), v.cuda(), 0.0, 0.1, x_dup=dup)


def test_no_cfg_branch_equals_the_duplicated_guidance_zero_form():
    """guidance_scale < 0 on the base model: the nb = 1 step gives the latents of the former cat([v, v]) mixed with
    guidance 0 (equal up to the sign of a zero)."""
    from r3g import ops
    from r3g.pipelines import HUNYUAN3D_2_CONFIG, Hunyuan3DDiTFlowMatchingPipeline
    cfg = dict(HUNYUAN3D_2_CONFIG, model=dict(HUNYUAN3D_2_CONFIG["model"], **MINI),
               vae=dict(HUNYUAN3D_2_CONFIG["vae"], num_latents=48, heads=2, width=128, num_decoder_layers=2))
    pipe = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=11, config=cfg, conditioner=None)
    torch.manual_seed(0)
    cond = {"main": torch.randn(1, 24, 96).cuda().half()}
    lat0 = torch.randn((1, 48, 64), generator=torch.manual_seed(99), dtype=torch.float16)
    steps = 6
    got = pipe(cond=cond, latents=lat0.clone(), num_inference_steps=steps, guidance_scale=-1.0, output_type="latent")
    sig = pipe.scheduler.step_sigmas()
    x = lat0.cuda().clone()
    for i, t in enumerate(pipe.scheduler.timesteps):
        ts = (t.to(torch.float16) / 1000).expand(1).cuda()
        v = pipe.model(x.clone(), ts, cond)
        ops.cfg_euler_step_(x, torch.cat([v, v]), 0.0, float((sig[i + 1] - sig[i]).half()))
    assert torch.equal(got, x)
    assert not torch.equal(got, lat0.cuda())


def test_guidance_timestep_embedding_against_reference_fixture(golden_dir):
    """The kernel's frequencies exp(-ln(1000) k / 128) come from the device expf, the fixture's from torch's CPU exp;
    the two may differ in the last float32 bits.  At guidance g the phase is 1000 g * freq, up to 10 000 rad, so a
    relative difference of a few 2^-24 moves it by up to ~2e-3 rad: hundreds of fp16 ulps for components near zero, where
    the time embedding's phases (<= 1000 rad) stay within ~1e-3.  Bound per element: |phase| * 2^-21 (four float32 ulps
    of the frequency) plus one fp16 ulp of the reference value."""
    from r3g import ops
    z = np.load(os.path.join(golden_dir, "dit_guidance_mini.npz"))
    ref = torch.from_numpy(z["gemb_out"])
    g16 = torch.from_numpy(z["gemb_g"])
    got = ops.timestep_embedding(g16.cuda(), 256, 1000.0, 1000.0).cpu()

    def line(h):        # fp16 bit patterns of finite values, sign-magnitude to a monotone integer line
        i = h.view(torch.int16).to(torch.int32)
        return torch.where(i < 0, -(i & 0x7FFF), i)
    ulps = (line(got) - line(ref)).abs()
    diff = (got.float() - ref.float()).abs()
    r = ref.float().abs().clamp_min(2.0 ** -14)
    ulp16 = 2.0 ** (torch.floor(torch.log2(r)) - 10)
    phase = (g16 * 1000).float()[:, None] * torch.exp(-np.log(1000.0) * torch.arange(128) / 128).repeat(1, 2)
    bound = phase * 2.0 ** -21 + ulp16
    print(f"guidance embedding, guidance {z['gemb_g'].tolist()}: {int((ulps > 0).sum())} of {ref.numel()} elements "
          f"differ; max {int(ulps.max())} fp16 ulp, max |diff| {diff.max().item():.3e}, max |diff| / bound "
          f"{(diff / bound).max().item():.3f}; elements > 1 ulp: {int((ulps > 1).sum())}")
    assert (diff <= bound).all()


def _mini_guided(golden_dir):
    from r3g.dit import Hunyuan3DDiT
    z = np.load(os.path.join(golden_dir, "dit_guidance_mini.npz"))
    m = Hunyuan3DDiT(guidance_embed=True, **MINI)
    import hy3d_distilled_ref as D
    m.load_state_dict(D.mini_state_dict(z["w_keys"], z["w_shapes"], int(z["w_seed"])))
    return z, m


def test_mini_guided_dit_against_reference_fixture_at_b2_and_b1(golden_dir):
    z, m = _mini_guided(golden_dir)
    x = torch.from_numpy(z["x"]).cuda().half()
    t = torch.from_numpy(z["t"]).cuda().half()
    c = torch.from_numpy(z["cond"]).cuda().half()
    g = torch.from_numpy(z["guidance"]).cuda().half()
    taps_ref = [torch.from_numpy(z[f"tap{i}"]) for i in range(4)]
    m.taps = []
    y = m(x, t, {"main": c}, guidance=g).float().cpu()
    for i, tp in enumerate(m.taps):
        assert rel_l2(tp.cpu(), taps_ref[i]) < 3e-3, i
    assert rel_l2(y, torch.from_numpy(z["y"])) < 1e-2
    yf = m(x, t, {"main": c}, guidance=g.flip(0)).float().cpu()
    assert rel_l2(yf, torch.from_numpy(z["y_flipped"])) < 1e-2
    for b in range(2):           # B = 1, the distilled pipeline's batch: gemv_kernel<1>, one-sample grouped GEMMs
        m.taps = []
        yb = m(x[b:b + 1], t[b:b + 1], {"main": c[b:b + 1]}, guidance=g[b:b + 1]).float().cpu()
        for i, tp in enumerate(m.taps):
            assert rel_l2(tp.cpu(), taps_ref[i][b:b + 1]) < 3e-3, (b, i)
        assert rel_l2(yb, torch.from_numpy(z["y"])[b:b + 1]) < 1e-2, b
    m.taps = None
    with pytest.raises(ValueError, match="guidance"):
        m(x, t, {"main": c})


@pytest.fixture(scope="module")
def turbo_pipe():
    from r3g.pipelines import HUNYUAN3D_2_TURBO_CONFIG, Hunyuan3DDiTFlowMatchingPipeline
    pipe = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=21, config=HUNYUAN3D_2_TURBO_CONFIG, conditioner=None)
    sd = {k: v.float().cuda() for k, v in pipe.model.reference_state_dict().items()}
    return pipe, sd


def test_full_guided_dit_b1_against_oracle(turbo_pipe):
    import hy3d_distilled_ref as D
    pipe, sd = turbo_pipe
    m = pipe.model
    torch.manual_seed(0)
    x = torch.randn(1, 3072, 64, device="cuda").half()
    c = torch.randn(1, 1370, 1536, device="cuda").half()
    t = torch.tensor([0.3994], device="cuda").half()
    g = torch.tensor([5.0], dtype=torch.float16, device="cuda")
    m.taps = []
    try:
        y = m(x, t, {"main": c}, guidance=g)
        taps_r3g = m.taps
    finally:
        m.taps = None
    taps = []
    ref = D.dit_forward(sd, x.float(), t.float(), c.float(), 16, 16, 32, guidance=g, taps=taps)
    assert len(taps_r3g) == len(taps) == 48
    errs = [rel_l2(a, b) for a, b in zip(taps_r3g, taps)]
    print(f"guided full-depth DiT, B = 1: per-block rel-L2 max {max(errs):.2e} (block {int(np.argmax(errs))}), "
          f"output {rel_l2(y, ref):.2e}")
    assert max(errs) < 1e-2, errs
    assert rel_l2(y, ref) < 2e-2


def test_distilled_pipeline_five_steps(turbo_pipe):
    import hy3d_distilled_ref as D
    import hy3d_ref as R
    pipe, sd = turbo_pipe
    torch.manual_seed(1)
    cond = {"main": torch.randn(1, 1370, 1536).cuda().half()}
    lat0 = torch.randn((1, 3072, 64), generator=torch.manual_seed(1234567), dtype=torch.float16)
    seen = []
    kw = dict(cond=cond, num_inference_steps=5, output_type="latent")
    pipe._graphs.entries.clear()
    out = pipe(latents=lat0.clone(), guidance_scale=5.0, callback=lambda i, t, o: seen.append((i, t, o)),
               callback_steps=1, **kw).clone()
    # one sample per step: the graph was captured for x [1, 3072, 64] and a [1, 1370, 1536] context
    assert [k[:2] for k in pipe._graphs.entries] == [((1, 3072, 64), (1, 1370, 1536))]
    pipe.use_cuda_graph = False
    try:
        eager = pipe(latents=lat0.clone(), guidance_scale=5.0, **kw)
    finally:
        pipe.use_cuda_graph = True
    assert torch.equal(out, eager), "CUDA-graph replay must reproduce eager launches bit for bit"
    other = pipe(latents=lat0.clone(), guidance_scale=3.5, **kw)
    assert not torch.equal(other, out), "the guidance scale must reach the model"
    ref = D.distilled_denoise_loop(sd, lat0.float().cuda(), cond["main"].float(), 16, 16, 32, 5, 5.0, 100,
                                   t_dtype=torch.float16)
    e = rel_l2(out, ref)
    print(f"latents after 5 distilled steps, 48 blocks: rel-L2 {e:.2e}")
    assert torch.isfinite(out).all() and e < 3e-2
    # the callback sees what ConsistencyFlowMatchEulerDiscreteScheduler.step returns
    sched = pipe.scheduler
    sig = sched.step_sigmas()
    assert [i for i, _, _ in seen] == list(range(5))
    g = torch.tensor([5.0], dtype=torch.float16, device="cuda")
    x = lat0.cuda()
    for i, t, o in seen:
        assert float(t) == float(sched.timesteps[i])
        v = pipe.model(x.clone(), (t.to(torch.float16) / 1000).expand(1).cuda(), cond, guidance=g)
        assert torch.equal(o.prev_sample.cpu(), R.flow_euler_step(x.cpu(), v.cpu(), sig[i], sig[i + 1])), i
        assert torch.equal(o.pred_original_sample, D.consistency_pred_original(x, v, sig[i].cuda())), i
        x = o.prev_sample
    assert torch.equal(x, out)


def test_distilled_pipeline_from_an_image_dense_and_flashvdm():
    """The turbo example's call (5 steps) from an RGBA crop: the stage's dense 257^3 decode, then FlashVDM at
    octree_resolution 380."""
    from PIL import Image
    from r3g.pipelines import HUNYUAN3D_2_TURBO_CONFIG, Hunyuan3DDiTFlowMatchingPipeline
    pipe = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=0, config=HUNYUAN3D_2_TURBO_CONFIG)
    rng = np.random.default_rng(5)
    yy, xx = np.mgrid[0:512, 0:512]
    rgba = np.zeros((512, 512, 4), np.uint8)
    rgba[..., :3] = rng.integers(0, 256, (512, 512, 3), dtype=np.uint8)
    rgba[..., 3] = ((((xx - 256) / 190.0) ** 2 + ((yy - 256) / 150.0) ** 2) <= 1.0) * 255
    img = Image.fromarray(rgba, "RGBA")
    dense = pipe(image=img, num_inference_steps=5, octree_resolution=256, num_chunks=16000,
                 generator=torch.manual_seed(1234567))[0]
    assert dense is not None and len(dense.faces) > 0 and len(dense.vertices) > 0
    pipe.enable_flashvdm()
    fast = pipe(image=img, num_inference_steps=5, octree_resolution=380, num_chunks=16000,
                generator=torch.manual_seed(1234567))[0]
    assert fast is not None and len(fast.faces) > 0 and len(fast.vertices) > 0
    print(f"image -> mesh in 5 distilled steps: dense 257^3 {len(dense.faces)} faces, FlashVDM 380 {len(fast.faces)} "
          f"faces; timings {pipe.timings}")
