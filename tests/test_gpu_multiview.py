"""GPU: Hunyuan3D-2mv on the r3g kernels.  The multi-view model is the 2.0 DiT on a context of V * 1370 rows, so the
kernels run at new shapes: the conditioner's DINOv2 forward on B * V images, the DiT's joint sequence of
3072 + 5480 = 8552 rows at V = 4, and the collapsed unconditional sample with 5479 copied text keys.

Tolerances are those of tests/test_gpu_models.py: the conditioner within rel-L2 5e-3 of transformers' Dinov2Model in
fp32; DiT hidden states after every block within rel-L2 3e-3 of the fp32 oracle, its output within 1e-2.  The view
embedding add, the collapsed unconditional forward, dict order and graph replay are compared bit for bit."""
import gc

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LT4 = 4 * 1370          # context rows of a four-view object


def rel_l2(a, b):
    a, b = a.float().flatten(), b.float().flatten()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def view_crop(seed, size=512):
    """An RGBA crop: noise RGB inside an ellipse whose shape depends on the seed."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:size, 0:size]
    ax, ay = rng.uniform(0.25, 0.4) * size, rng.uniform(0.2, 0.35) * size
    rgba = np.zeros((size, size, 4), np.uint8)
    rgba[..., :3] = rng.integers(0, 256, (size, size, 3), dtype=np.uint8)
    rgba[..., 3] = ((((xx - size / 2) / ax) ** 2 + ((yy - size / 2) / ay) ** 2) <= 1.0) * 255
    return Image.fromarray(rgba, "RGBA")


def test_mv_conditioner_on_r3g_kernels_against_the_hf_module():
    """DINOv2-g width (1536, 24 heads of 64, SwiGLU 4096) on B * V = 4 images at 518 px, four layers; then the view
    embedding add, which must be torch's fp16 add of the table's rows to the same hidden states."""
    from r3g.conditioner import DINOV2_GIANT, DinoImageEncoderMV
    cfg = dict(DINOV2_GIANT, num_hidden_layers=4)
    torch.manual_seed(0)
    enc = DinoImageEncoderMV(config=cfg, image_size=518, view_num=4, device="cuda", dtype=torch.float16)
    assert enc.backend == "r3g"
    with torch.no_grad():
        for n, p_ in enc.model.named_parameters():
            if "lambda1" in n:
                p_.copy_(0.3 + 0.2 * torch.rand_like(p_))
            elif "norm" in n and n.endswith("weight"):
                p_.copy_(1 + 0.2 * torch.randn_like(p_))
    img = torch.rand(1, 4, 3, 512, 512) * 2 - 1
    idxs = [(0, 1, 2, 3)]
    got = enc(img, view_idxs=idxs)
    assert got.shape == (1, LT4, 1536) and got.dtype == torch.float16
    # the add, bit for bit: r3g hidden states + the fp16 table rows
    px = enc._transform(((img.view(4, 3, 512, 512) + 1) / 2).cuda().half())
    hid = enc._forward_r3g(px).view(1, 4, 1370, 1536)
    tab16 = torch.from_numpy(enc.view_table).cuda().half()
    assert torch.equal(got, (hid + tab16[None, :, None, :]).view(1, LT4, 1536))
    other = enc(img, view_idxs=[(3, 2, 1, 0)])
    assert torch.equal(other, (hid + tab16.flip(0)[None, :, None, :]).view(1, LT4, 1536))
    # against the HF module in fp32 on the same weights, with the float32 table
    ref_model = type(enc.model)(enc.model.config).to("cuda").float()
    ref_model.load_state_dict({k: v.float() for k, v in enc.model.state_dict().items()})
    with torch.no_grad():
        ref = ref_model(px.float()).last_hidden_state.view(1, 4, 1370, 1536)
    ref = (ref + torch.from_numpy(enc.view_table).cuda()[None, :, None, :]).view(1, LT4, 1536)
    e = rel_l2(got, ref)
    print(f"MV conditioner, 4 views at DINOv2-g width: rel-L2 {e:.2e}")
    assert e < 5e-3, e
    u = enc.unconditional_embedding(1, view_idxs=idxs)
    assert u.shape == (1, LT4, 1536) and u.dtype == torch.float16 and not u.any()


def test_dit_full_width_blocks_at_the_four_view_context():
    """hidden 1024 / 16 heads, Lt = 5480, L = 8552, 1 double + 2 single blocks, B = 2, against the fp32 oracle."""
    import hy3d_ref as R
    from r3g.dit import Hunyuan3DDiT
    m = Hunyuan3DDiT(depth=1, depth_single_blocks=2).init_random(seed=3)
    m.taps = []
    torch.manual_seed(0)
    x = torch.randn(2, 3072, 64, device="cuda").half()
    c = torch.randn(2, LT4, 1536, device="cuda").half()
    t = torch.tensor([0.5102, 0.5102], device="cuda").half()
    y = m(x, t, {"main": c})
    sd = {k: v.float().cuda() for k, v in m.reference_state_dict().items()}
    taps = []
    ref = R.dit_forward(sd, x.float(), t.float(), c.float(), 16, 1, 2, taps=taps)
    assert len(m.taps) == len(taps) == 3 and m.taps[0].shape == (2, 3072 + LT4, 1024)
    for i, (a, b) in enumerate(zip(m.taps, taps)):
        e = rel_l2(a, b)
        print(f"Lt = {LT4}: tap {i} rel-L2 {e:.2e}")
        assert e < 3e-3, f"tap {i}: rel L2 {e}"
    assert rel_l2(y, ref) < 1e-2


@pytest.fixture(scope="module")
def full_dit():
    from r3g.dit import Hunyuan3DDiT
    return Hunyuan3DDiT().init_random(seed=21)


def test_full_depth_collapsed_equals_full_at_the_four_view_context(full_dit):
    """The unconditional sample's zero 5480-row context collapses to one row (3073 live query rows, 5479 copied keys);
    the output must be the full forward's bit for bit, for the CFG pair and for the lone samples."""
    m = full_dit
    torch.manual_seed(0)
    x = torch.randn(2, 3072, 64, device="cuda").half()
    c = torch.cat([torch.randn(1, LT4, 1536, device="cuda"), torch.zeros(1, LT4, 1536, device="cuda")]).half()
    t = torch.tensor([0.3469, 0.3469], device="cuda").half()
    full = m(x, t, {"main": c}).clone()
    coll = m(x, t, {"main": c}, uncond_txt_shared=True).clone()
    assert torch.equal(coll, full)
    lone_c = m(x[:1].contiguous(), t[:1], {"main": c[:1].contiguous()}).clone()
    lone_u = m(x[1:].contiguous(), t[1:], {"main": c[1:].contiguous()}, uncond_txt_shared=True).clone()
    assert torch.equal(lone_c, full[:1]) and torch.equal(lone_u, full[1:])


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def test_pipeline_three_views_order_invariant_and_graph_equals_eager():
    from r3g.pipelines import HUNYUAN3D_2MV_CONFIG, Hunyuan3DDiTFlowMatchingPipeline
    _free()
    pipe = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=0, config=HUNYUAN3D_2MV_CONFIG)
    views = {tag: view_crop(40 + i) for i, tag in enumerate(("front", "left", "back"))}
    kw = dict(num_inference_steps=10, octree_resolution=256, num_chunks=16000)
    mesh = pipe(image=views, generator=torch.manual_seed(1234567), **kw)[0]
    assert mesh is not None and len(mesh.faces) > 0 and len(mesh.vertices) > 0
    # one graph for the CFG pair at the three-view context, on the collapsed unconditional path
    keys = list(pipe._graphs.entries)
    assert len(keys) == 1 and keys[0][1] == (2, 3 * 1370, 1536) and keys[0][2] is True
    reordered = {tag: views[tag] for tag in ("back", "left", "front")}
    again = pipe(image=reordered, generator=torch.manual_seed(1234567), **kw)[0]
    assert np.array_equal(again.vertices, mesh.vertices) and np.array_equal(again.faces, mesh.faces)
    # another view count is another context shape, so another graph
    two = pipe(image={"right": views["front"], "front": views["back"]}, generator=torch.manual_seed(7),
               num_inference_steps=2, output_type="latent")
    assert two.shape == (1, 3072, 64) and len(pipe._graphs.entries) == 2
    # graph replay against the eager launches
    lat = {}
    for graph in (True, False):
        pipe.use_cuda_graph = graph
        lat[graph] = pipe(image=views, generator=torch.manual_seed(1234567), num_inference_steps=10,
                          output_type="latent").clone()
    assert torch.isfinite(lat[True]).all() and torch.equal(lat[True], lat[False])
    print(f"2mv, 3 views: {len(mesh.faces)} faces; timings {pipe.timings}")
    del pipe
    _free()


def test_turbo_pipeline_four_views_with_flashvdm():
    from r3g.pipelines import HUNYUAN3D_2MV_TURBO_CONFIG, Hunyuan3DDiTFlowMatchingPipeline
    _free()
    pipe = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=0, config=HUNYUAN3D_2MV_TURBO_CONFIG)
    views = {tag: view_crop(50 + i) for i, tag in enumerate(("front", "left", "back", "right"))}
    pipe.enable_flashvdm()
    mesh = pipe(image=views, num_inference_steps=5, octree_resolution=380, num_chunks=16000,
                generator=torch.manual_seed(1234567))[0]
    assert mesh is not None and len(mesh.faces) > 0 and len(mesh.vertices) > 0
    keys = list(pipe._graphs.entries)
    assert len(keys) == 1 and keys[0][0] == (1, 3072, 64) and keys[0][1] == (1, LT4, 1536)   # no CFG: one sample
    print(f"2mv-turbo, 4 views, FlashVDM 380: {len(mesh.faces)} faces; timings {pipe.timings}")
    del pipe
    _free()
