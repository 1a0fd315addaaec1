"""GPU: the pipeline mirror end to end on a reduced configuration (real kernels, small widths) against the
fp32 oracle loop, CUDA-graph replay vs eager launch, and mesh extraction against the CPU marching-cubes oracle."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MINI = dict(
    model=dict(in_channels=64, context_in_dim=96, hidden_size=128, num_heads=2, depth=2, depth_single_blocks=2),
    vae=dict(num_latents=48, embed_dim=64, num_freqs=8, include_pi=False, heads=2, width=128, num_decoder_layers=2,
             qkv_bias=False, qk_norm=True, scale_factor=0.999),
    scheduler=dict(num_train_timesteps=1000),
    image_processor=dict(size=512, border_ratio=0.15),
)


def make_pipe():
    from r3g.pipelines import Hunyuan3DDiTFlowMatchingPipeline
    return Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=11, config=MINI, conditioner=None)


def test_denoise_loop_against_oracle_and_graph_equals_eager():
    import hy3d_ref as R
    pipe = make_pipe()
    torch.manual_seed(0)
    cond = {"main": torch.cat([torch.randn(1, 24, 96), torch.zeros(1, 24, 96)]).cuda().half()}
    gen = torch.manual_seed(1234567)
    lat0 = torch.randn((1, 48, 64), generator=gen, dtype=torch.float16)
    outs = {}
    for graph in (False, True):
        pipe.use_cuda_graph = graph
        outs[graph] = pipe(cond=cond, latents=lat0.clone(), num_inference_steps=6, guidance_scale=5.0,
                           output_type="latent")
    assert torch.equal(outs[False], outs[True]), "CUDA-graph replay must reproduce eager launches bit for bit"
    sd = {k: v.float() for k, v in pipe.model.reference_state_dict().items()}
    ref = R.denoise_loop(sd, lat0.float(), cond["main"].float().cpu(), 2, 2, 2, 6, 5.0, t_dtype=torch.float16)
    err = ((outs[True].float().cpu() - ref).norm() / ref.norm()).item()
    assert err < 2e-2, f"latents after 6 CFG steps: rel L2 {err}"
    # the same seed through the generator path gives the same latents as the explicit draw
    again = pipe(cond=cond, generator=torch.manual_seed(1234567), num_inference_steps=6, guidance_scale=5.0,
                 output_type="latent")
    assert torch.equal(again, outs[True])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_graphs_on_a_device_that_is_not_current():
    """Models on cuda:1 with cuda:0 current: graph capture and replay follow the inputs' device."""
    from r3g.pipelines import Hunyuan3DDiTFlowMatchingPipeline
    from r3g.vggt_heads import CameraHeadR3G, random_state_dict
    torch.cuda.set_device(0)
    dev = torch.device("cuda:1")
    sd = random_state_dict(7, embed_dim=128, depth=1, vit_depth=1, trunk_depth=2, features=32,
                           out_channels=(32, 64, 128, 128), img_size=56)
    head = CameraHeadR3G({k: v for k, v in sd.items() if k.startswith("camera_head.")}, trunk_depth=2, num_heads=2,
                         device=dev)
    toks = [torch.randn(1, 2, 7, 256, device=dev)]
    graph = head(toks)
    head.use_cuda_graph = False
    assert all(torch.equal(a, b) for a, b in zip(graph, head(toks)))
    pipe = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=11, config=MINI, conditioner=None, device=dev)
    cond = {"main": torch.cat([torch.randn(1, 24, 96), torch.zeros(1, 24, 96)]).to(dev).half()}
    lat0 = torch.randn((1, 48, 64), generator=torch.manual_seed(1234567), dtype=torch.float16)
    outs = {}
    for use_graph in (False, True):
        pipe.use_cuda_graph = use_graph
        outs[use_graph] = pipe(cond=cond, latents=lat0.clone(), num_inference_steps=6, guidance_scale=5.0,
                               output_type="latent")
    assert outs[True].device == dev and torch.equal(outs[False], outs[True])
    assert torch.cuda.current_device() == 0


def test_mesh_output_matches_cpu_marching_cubes_on_the_same_grid():
    import mc as omc
    pipe = make_pipe()
    cond = {"main": torch.cat([torch.randn(1, 24, 96), torch.zeros(1, 24, 96)]).cuda().half()}
    out = pipe(cond=cond, generator=torch.manual_seed(7), num_inference_steps=4, octree_resolution=24,
               output_type="mesh", mc_level=0.0)
    grid = pipe.last_grid[0].cpu().numpy()
    try:
        ov, of = omc.marching_cubes(grid, 0.0, bounds=[-1.01] * 3 + [1.01] * 3)
    except (ValueError, RuntimeError):
        assert out[0] is None
        return
    assert np.array_equal(out[0].mesh_v, ov) and np.array_equal(out[0].mesh_f, of)
    tri = pipe(cond=cond, generator=torch.manual_seed(7), num_inference_steps=4, octree_resolution=24)[0]
    assert np.array_equal(np.asarray(tri.faces), of[:, ::-1])


def test_surface_extractor_swallows_failures_like_the_reference():
    from r3g.vae import MCSurfaceExtractor
    ex = MCSurfaceExtractor()
    flat = torch.zeros(1, 9, 9, 9, device="cuda")
    assert ex(flat, mc_level=0.0, bounds=1.01, octree_resolution=8) == [None]
