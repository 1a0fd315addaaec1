"""GPU: dual marching cubes (ops.dual_marching_cubes, R3G_MC_DUAL) through the C ABI, bit-exact against the CPU oracle
(oracle/dmc_oracle.c: float32 vertices, integer faces, order), and the 'dmc' surface extractor of the pipeline."""
import numpy as np
import pytest
import torch

from test_dmc_oracle import with_nans
from test_gpu_mc import _vols
from test_mc_oracle import check_closed_manifold, random_field

pytestmark = pytest.mark.gpu


def _cuda_dmc(vol):
    from r3g import ops
    v, f = ops.dual_marching_cubes(torch.from_numpy(vol).cuda())
    assert v.dtype == torch.float32 and f.dtype == torch.int32 and v.is_cuda and f.is_cuda
    return v.cpu().numpy(), f.cpu().numpy()


@pytest.mark.parametrize("name,vol", list(_vols()) + [("nan_random_field", with_nans(random_field(33, 4), 4)),
                                                      ("nan_noise", with_nans(np.random.default_rng(9).standard_normal(
                                                          (16, 17, 18)).astype(np.float32), 9, 0.1))])
def test_dmc_bit_exact(name, vol):
    import dmc as odmc
    ov, of = odmc.dual_marching_cubes(vol)
    v, f = _cuda_dmc(vol)
    assert np.array_equal(f, of), f"{name}: faces differ"
    assert np.array_equal(v, ov, equal_nan=True), f"{name}: vertex positions differ"


def test_dmc_unaligned_grid_pointer():
    import dmc as odmc
    from r3g import ops
    vol = random_field(33, 5)
    ov, of = odmc.dual_marching_cubes(vol)
    flat = torch.empty(vol.size + 1, device="cuda")
    g = flat[1:].view(vol.shape)
    g.copy_(torch.from_numpy(vol))
    assert g.data_ptr() % 16 != 0 and g.is_contiguous()
    v, f = ops.dual_marching_cubes(g)
    assert np.array_equal(f.cpu().numpy(), of) and np.array_equal(v.cpu().numpy(), ov)


def test_dmc_no_surface_and_argument_checks():
    import ctypes as C
    from r3g import _abi, ops
    from r3g.vae import DMCSurfaceExtractor
    with pytest.raises(RuntimeError):
        ops.dual_marching_cubes(torch.zeros(5, 5, 5, device="cuda"))
    assert DMCSurfaceExtractor()(torch.zeros(1, 9, 9, 9, device="cuda"), mc_level=0.0, bounds=1.01,
                                 octree_resolution=8) == [None]
    # a volume that lies entirely above the level has no crossed cell either (no level-range error in dual mode)
    assert DMCSurfaceExtractor()(torch.ones(1, 9, 9, 9, device="cuda"), octree_resolution=8) == [None]
    g = torch.from_numpy(random_field(9, 1)).cuda()
    ops.dual_marching_cubes(g)                                  # leaves the count of g in the workspace
    ws = ops._workspace("mc", g.device, 0)
    verts = torch.empty(4096, 3, device="cuda")
    faces = torch.empty(4096, 3, device="cuda", dtype=torch.int32)
    bounds = (C.c_double * 6)(*([-1.0] * 3 + [1.0] * 3))
    for method, bptr in ((_abi.R3G_MC_DUAL, C.cast(bounds, C.c_void_p)), (2, C.c_void_p(0))):
        with pytest.raises(_abi.R3GError) as e:
            ops._launch("mc_extract", g, g, 9, 9, 9, 0.0, method, bptr, ws, ws.numel(), verts, faces)
        assert e.value.code == _abi.R3G_E_INVALID


def test_dmc_257_torus_closed_and_deterministic():
    from r3g import ops
    n = 257
    ax = torch.linspace(-1.01, 1.01, n, device="cuda")
    x, y, z = torch.meshgrid(ax, ax, ax, indexing="ij")
    vol = (0.25 - torch.sqrt((torch.sqrt(x * x + y * y) - 0.6) ** 2 + z * z)).contiguous()
    v, f = ops.dual_marching_cubes(vol)
    assert check_closed_manifold(v.cpu().numpy(), f.cpu().numpy()) == 0
    v2, f2 = ops.dual_marching_cubes(vol)
    assert torch.equal(v, v2) and torch.equal(f, f2)


def _centred_oracle(grid):
    import dmc as odmc
    from r3g.vae import center_vertices
    ov, of = odmc.dual_marching_cubes(grid)
    return center_vertices(torch.from_numpy(ov)).numpy(), of


def test_pipeline_mc_algo_dmc_equals_the_oracle():
    from test_gpu_pipeline import make_pipe
    pipe = make_pipe()
    cond = {"main": torch.cat([torch.randn(1, 24, 96, generator=torch.manual_seed(3)), torch.zeros(1, 24, 96)]).cuda().half()}
    out = pipe(cond=cond, generator=torch.manual_seed(7), num_inference_steps=4, octree_resolution=24,
               output_type="mesh", mc_algo="dmc")
    grid = pipe.last_grid[0].float().cpu().numpy()
    try:
        ov, of = _centred_oracle(grid)
    except RuntimeError:
        assert out[0] is None
        return
    print(f"\npipeline dmc at octree 24: V={len(ov)} F={len(of)}")
    assert out[0] is not None and np.array_equal(out[0].mesh_v, ov) and np.array_equal(out[0].mesh_f, of)
    tri = pipe(cond=cond, generator=torch.manual_seed(7), num_inference_steps=4, octree_resolution=24,
               mc_algo="dmc")[0]
    assert np.array_equal(np.asarray(tri.faces), of[:, ::-1])


def test_flashvdm_mc_algo_dmc_equals_the_oracle_on_its_nan_grid():
    from r3g.vae import DMCSurfaceExtractor, FlashVDMVolumeDecoding
    from test_gpu_pipeline import make_pipe
    pipe = make_pipe()
    pipe.enable_flashvdm(mc_algo="dmc")
    assert isinstance(pipe.vae.volume_decoder, FlashVDMVolumeDecoding)
    assert isinstance(pipe.vae.surface_extractor, DMCSurfaceExtractor)
    cond = {"main": torch.cat([torch.randn(1, 24, 96, generator=torch.manual_seed(3)), torch.zeros(1, 24, 96)]).cuda().half()}
    out = pipe(cond=cond, generator=torch.manual_seed(7), num_inference_steps=4, octree_resolution=128,
               output_type="mesh")
    g = pipe.last_grid[0]
    assert g.dtype == torch.float16
    grid = g.float().cpu().numpy()
    print(f"\nFlashVDM grid {grid.shape}: {np.isnan(grid).mean():.3f} NaN")
    try:
        ov, of = _centred_oracle(grid)
    except RuntimeError:
        assert out[0] is None
        return
    assert out[0] is not None
    assert np.array_equal(out[0].mesh_v, ov, equal_nan=True) and np.array_equal(out[0].mesh_f, of)
    # before centring: a crossing next to a NaN point is NaN, the others are finite and equal the oracle's.  (The
    # reference's center_vertices takes min / max over all vertices, so one NaN vertex makes every centred vertex NaN.)
    import dmc as odmc
    from r3g import ops
    uv, uf = ops.dual_marching_cubes(g.float())
    rv, rf = odmc.dual_marching_cubes(grid)
    nan = np.isnan(rv).any(1)
    print(f"FlashVDM dmc: V={len(rv)} F={len(rf)}, {nan.sum()} vertices with a NaN crossing")
    assert np.array_equal(uv.cpu().numpy(), rv, equal_nan=True) and np.array_equal(uf.cpu().numpy(), rf)
    assert (~nan).any()


def test_floater_removal_and_face_reduction_on_the_dmc_torus():
    from r3g import ops
    from r3g.postprocessors import FaceReducerR3G, FloaterRemover
    n = 257
    ax = torch.linspace(-1.01, 1.01, n, device="cuda")
    x, y, z = torch.meshgrid(ax, ax, ax, indexing="ij")
    vol = (0.25 - torch.sqrt((torch.sqrt(x * x + y * y) - 0.6) ** 2 + z * z)).contiguous()
    v, f = ops.dual_marching_cubes(vol)
    v, f = FloaterRemover()((v, f))
    target = 40000
    assert len(f) > target
    vr, fr = FaceReducerR3G()((v, f), max_facenum=target)
    assert vr.is_cuda and len(fr) in (target, target - 1)
    assert check_closed_manifold(vr.cpu().numpy(), fr.cpu().numpy()) == 0
