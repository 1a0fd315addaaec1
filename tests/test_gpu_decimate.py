"""GPU: r3g_mesh_decimate (FaceReducerR3G) against its numpy mirror, bit for bit, and the properties of the reduced meshes
at the sizes stage 3 produces."""
import json
import os
import struct
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from test_decimate_oracle import CASES, FIELDS, check_reduced, mc_mesh, sdf_scene3, sdf_sphere, topology

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(v, f, target):
    from r3g import ops
    vo, fo, rounds = ops.mesh_decimate(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), target)
    return vo.cpu().numpy(), fo.cpu().numpy(), rounds


@pytest.mark.parametrize("kind, n, targets, bound", CASES, ids=[c[0] for c in CASES])
def test_cuda_equals_the_mirror_bit_for_bit(kind, n, targets, bound):
    import decimate as odec
    v0, f0 = mc_mesh(kind, n)
    for target in targets + (0,):
        v, f, r = _run(v0, f0, target)
        ov, of, orr = odec.decimate(v0, f0, target)
        assert r == orr and np.array_equal(f, of), (kind, target, r, orr, len(f), len(of))
        assert np.array_equal(v.view(np.uint32), ov.view(np.uint32)), (kind, target)
        v2, f2, _ = _run(v0, f0, target)                 # deterministic: a second run is the same
        assert np.array_equal(v2.view(np.uint32), v.view(np.uint32)) and np.array_equal(f2, f)


def test_257_sphere_to_40000_equals_the_mirror():
    import decimate as odec
    v0, f0 = mc_mesh("sphere", 257)
    assert len(f0) > 200000
    v, f, r = _run(v0, f0, 40000)
    t = time.time()
    ov, of, orr = odec.decimate(v0, f0, 40000)
    print(f"\nmirror at 257^3: {time.time() - t:.1f} s, {orr} rounds")
    assert r == orr and np.array_equal(f, of) and np.array_equal(v.view(np.uint32), ov.view(np.uint32))
    err = check_reduced(v0, f0, v, f, 40000, sdf_sphere, 0.002)
    print(f"sphere 257^3: {len(f0)} -> {len(f)} faces in {r} rounds, max |sdf| {err:.3e}")


def test_257_scene_to_40000_keeps_the_surface():
    v0, f0 = mc_mesh("scene3", 257)
    v, f, r = _run(v0, f0, 40000)
    err = check_reduced(v0, f0, v, f, 40000, sdf_scene3, 0.004)
    print(f"\nscene 257^3: {len(f0)} -> {len(f)} faces in {r} rounds, max |sdf| {err:.3e}")


def test_noise_mesh_terminates_with_the_invariants():
    """test_components_on_a_large_noise_mesh's 129^3 noise mesh: thousands of components, so 40 000 faces is out of
    reach; the rounds stop at the smallest mesh the rules allow, topology intact."""
    from r3g import ops
    from r3g.postprocessors import FaceReducerR3G
    g = torch.Generator(device="cuda").manual_seed(0)
    grid = torch.randn(129, 129, 129, device="cuda", generator=g)
    v0, f0 = ops.marching_cubes(grid, 0.0)
    t = time.time()
    v, f = FaceReducerR3G()((v0, f0))
    torch.cuda.synchronize()
    print(f"\nnoise 129^3: {len(f0)} -> {len(f)} faces in {time.time() - t:.2f} s")
    assert v.is_cuda and f.is_cuda and 40000 < len(f) < len(f0)
    v0n, f0n, vn, fn = v0.cpu().numpy(), f0.cpu().numpy(), v.cpu().numpy(), f.cpu().numpy()
    chi0, comp0, loops0, _, twice0, over0 = topology(v0n, f0n)
    chi, comp, loops, _, twice, over = topology(vn, fn)
    assert (chi, comp, loops) == (chi0, comp0, loops0)
    assert twice <= twice0 and over <= over0
    assert ((fn[:, 0] != fn[:, 1]) & (fn[:, 1] != fn[:, 2]) & (fn[:, 0] != fn[:, 2])).all()
    assert len(np.unique(fn)) == len(vn)


def test_input_forms_devices_and_bad_indices():
    import decimate as odec
    from r3g import _abi, ops
    from r3g.postprocessors import FaceReducerR3G
    from r3g.vae import Latent2MeshOutput
    v0, f0 = mc_mesh("torus", 41)
    ov, of, _ = odec.decimate(v0, f0, 1500)
    red = FaceReducerR3G()
    out = red(Latent2MeshOutput(mesh_v=v0, mesh_f=f0), max_facenum=1500)
    assert isinstance(out, Latent2MeshOutput) and np.array_equal(out.mesh_v, ov) and np.array_equal(out.mesh_f, of)

    class Obj:
        def __init__(self, vertices, faces):
            self.vertices, self.faces = vertices, faces
    o = red(Obj(v0, f0.astype(np.int64)), max_facenum=1500)
    assert isinstance(o, Obj) and np.array_equal(o.faces, of)
    vt, ft = red((torch.from_numpy(v0).cuda(), torch.from_numpy(f0).cuda()), max_facenum=1500)
    assert vt.is_cuda and ft.is_cuda and np.array_equal(ft.cpu().numpy(), of)
    vn, fn = red((v0, f0), max_facenum=1500)
    assert isinstance(vn, np.ndarray) and np.array_equal(vn, ov)
    small = (v0, f0)
    assert red(small, max_facenum=len(f0) + 1) is small
    if torch.cuda.device_count() > 1:
        v1, f1 = red((torch.from_numpy(v0).to("cuda:1"), torch.from_numpy(f0).to("cuda:1")), max_facenum=1500)
        assert v1.device == torch.device("cuda:1") and np.array_equal(f1.cpu().numpy(), of)
    for bad in (len(v0), -1):
        fb = f0.copy()
        fb[7, 1] = bad
        with pytest.raises(_abi.R3GError) as e:
            ops.mesh_decimate(torch.from_numpy(v0).cuda(), torch.from_numpy(fb).cuda(), 100)
        assert e.value.code == _abi.R3G_E_INVALID
    with pytest.raises(ValueError):
        ops.mesh_decimate(torch.from_numpy(v0).cuda(), torch.from_numpy(f0).cuda(), -1)


def _glb_faces(path):
    data = open(path, "rb").read()
    n = struct.unpack_from("<I", data, 12)[0]
    gltf = json.loads(data[20:20 + n])
    return gltf["accessors"][gltf["meshes"][0]["primitives"][0]["indices"]]["count"] // 3


def test_stage3_twin_writes_reduced_meshes(tmp_path):
    """The stage script at octree 256: the raw meshes exceed 40 000 faces and the .glb files hold the reduced meshes.
    Random weights give a noise-like field whose meshes fall apart into thousands of small components, each of which
    keeps at least a tetrahedron, so the reduction stops above 40 000 faces; the count reaches 40 000 where it can
    (test_257_*)."""
    import re
    import yaml
    sys.path.insert(0, ROOT)
    from bench import synthetic_crop
    inp, out = tmp_path / "in", tmp_path / "out"
    inp.mkdir()
    out.mkdir()
    for name, seed in (("chair__1.png", 1), ("table__2.png", 2)):
        synthetic_crop(seed).save(inp / name)
    cfg = dict(use_banana=False, input_folder_hy=str(inp), output_folder_hy=str(out), num_inf_steps_hy=3,
               octree_resolution_hy=256, num_chunks_hy=16000, seed=1234567, mini=False)
    (tmp_path / "config.yaml").write_text(yaml.safe_dump(cfg))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "stages", "2d_to_3d_models", "run.py"), "--config",
                        str(tmp_path / "config.yaml"), "--random-weights"], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    lines = {m.group(1): (int(m.group(2)), int(m.group(3))) for m in
             re.finditer(r"\] (\S+): \d+ vertices, (\d+) faces \(reduced from (\d+)\)", r.stdout)}
    print("\n" + "\n".join(f"{k}: {raw} -> {red} faces" for k, (red, raw) in lines.items()))
    assert set(lines) == {"chair__1", "table__2"}
    for stem, (reduced, raw) in lines.items():
        assert raw > 40000, (stem, raw)
        assert reduced < raw
        assert _glb_faces(out / stem / f"{stem}.glb") == reduced
