"""CPU: host-side logic of the pipeline mirror that needs no GPU (mesh export, scheduler mirror, image processor,
stage-script helpers)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_simple_mesh_glb_roundtrip(tmp_path):
    import json
    import struct
    from r3g.pipelines import SimpleMesh
    v = np.random.rand(5, 3).astype(np.float32)
    f = np.array([[0, 1, 2], [2, 3, 4]], np.int32)
    p = SimpleMesh(v, f).export(str(tmp_path / "a.glb"))
    raw = open(p, "rb").read()
    magic, ver, total = struct.unpack("<4sII", raw[:12])
    assert magic == b"glTF" and ver == 2 and total == len(raw)
    jl = struct.unpack("<I", raw[12:16])[0]
    doc = json.loads(raw[20:20 + jl])
    off = 20 + jl + 8
    idx = np.frombuffer(raw[off:off + 24], "<u4").reshape(2, 3)
    pos = np.frombuffer(raw[off + 24:off + 24 + 60], "<f4").reshape(5, 3)
    assert np.array_equal(idx, f) and np.array_equal(pos, v) and doc["accessors"][1]["count"] == 5


def test_scheduler_mirror_matches_reference_fixture(golden_dir):
    from r3g.scheduler import FlowMatchEulerDiscreteScheduler
    z = np.load(os.path.join(golden_dir, "scheduler.npz"))
    sch = FlowMatchEulerDiscreteScheduler(num_train_timesteps=1000)
    for n in (1, 5, 50):
        sch.set_timesteps(sigmas=np.linspace(0, 1, n))
        assert np.array_equal(sch.timesteps.numpy(), z[f"timesteps_{n}"])
        assert np.array_equal(sch.sigmas.numpy(), z[f"sigmas_{n}"])
    sch.set_timesteps(sigmas=np.linspace(0, 1, 5))
    x = torch.from_numpy(z["euler_x"][0])
    for i, t in enumerate(sch.timesteps[:3]):
        x = sch.step(torch.from_numpy(z["euler_v"][i]), t, x).prev_sample
        assert np.array_equal(x.numpy(), z["euler_x"][i + 1])
    with pytest.raises(ValueError):
        sch.step(torch.zeros(1), 3, torch.zeros(1))


def _reference_checks(golden_dir):
    return np.load(os.path.join(golden_dir, "reference_checks.npz"))


def _sha(a):
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def test_image_processor_against_reference_when_available(golden_dir):
    """ImageProcessorV2 (preprocessors.py) against the reference's output on the same seeded RGBA image, stored as a
    sha256 of the image / mask tensors plus a seeded sample (oracle/make_reference_checks.py)."""
    import make_reference_checks as mrc
    from r3g.preprocessors import ImageProcessorV2
    z = _reference_checks(golden_dir)
    a = ImageProcessorV2(512, 0.15)(mrc.imgproc_input())
    img, mask = a["image"].numpy(), a["mask"].numpy()
    assert img.shape == (1, 3, 512, 512) and mask.shape == (1, 1, 512, 512)
    assert tuple(z["imgproc_image_shape"]) == img.shape and tuple(z["imgproc_mask_shape"]) == mask.shape
    assert str(img.dtype) == str(z["imgproc_image_dtype"]) and str(mask.dtype) == str(z["imgproc_mask_dtype"])
    assert np.array_equal(img.reshape(-1)[mrc.sample_idx(img.size)], z["imgproc_image_sample"])
    assert _sha(img) == str(z["imgproc_image_sha256"]) and _sha(mask) == str(z["imgproc_mask_sha256"])


def test_stage3_twin_file_contract(tmp_path, monkeypatch):
    """The stage-3 twin's host helpers: config loading, name filter, output clearing (no GPU work here)."""
    sys.path.insert(0, os.path.join(ROOT, "stages", "2d_to_3d_models"))
    import importlib
    run = importlib.import_module("run")
    d = tmp_path / "out"
    (d / "old").mkdir(parents=True)
    (d / "old" / "x.glb").write_bytes(b"1")
    (d / "stale.txt").write_text("x")
    run.clear_output_directory(str(d))
    assert os.listdir(d) == []
    cfg = tmp_path / "c.yaml"
    cfg.write_text("num_inf_steps_hy: 50\noctree_resolution_hy: 256\nuse_banana: false\n")
    assert run.load_config(str(cfg))["octree_resolution_hy"] == 256


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` (the CPU oracle port on the host cores) prints one JSON line with the contract's keys;
    under torchrun only rank 0 prints."""
    import json
    import subprocess
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-500:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["unit"] == "objects/s" and line["higher_is_better"] is True
    assert line["metric"].startswith("objects->mesh/sec") and line["value"] > 0 and line["steps"] == 1
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
    assert line["e2e"] == {"value": line["value"], "unit": "objects/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    r1 = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                        capture_output=True, text=True, timeout=60, cwd=ROOT, env=dict(os.environ, RANK="1", WORLD_SIZE="2"))
    assert r1.returncode == 0 and r1.stdout.strip() == ""


def test_conditioner_mirror_against_reference_when_available(golden_dir):
    """Row a2: DinoImageEncoder (conditioner.py:57-131) -- value-range shift, Resize(bilinear, antialias) + CenterCrop +
    Normalize, HF Dinov2Model, cls token kept; zeros as the unconditional embedding.  The reference's small random model
    and its outputs on seeded inputs are stored (oracle/make_reference_checks.py)."""
    import make_reference_checks as mrc
    from r3g.conditioner import DinoImageEncoder, SingleImageEncoder
    z = _reference_checks(golden_dir)
    mine = DinoImageEncoder(config=mrc.COND_CFG, use_cls_token=True, image_size=56, device="cpu", dtype=torch.float32)
    mine.model.load_state_dict({k[len("cond_w:"):]: torch.from_numpy(z[k]) for k in z.files if k.startswith("cond_w:")})
    for i, (shape, img) in enumerate(zip(mrc.COND_SHAPES, mrc.cond_inputs())):
        a, b = mine(img), torch.from_numpy(z[f"cond_out{i}"])
        assert a.shape == b.shape == (shape[0], 17, 32)
        assert torch.allclose(a, b, atol=1e-5, rtol=1e-5), (a - b).abs().max()
    u = SingleImageEncoder(mine).unconditional_embedding(2)["main"]
    assert u.shape == (2, 17, 32) and not u.any() and torch.equal(u, torch.from_numpy(z["cond_uncond"]))


def test_near_surface_mask_against_reference_when_available(golden_dir):
    """extract_near_surface_volume_fn (volume_decoders.py:29-119): the point selection of the FlashVDM levels, against
    the reference's masks on the same seeded volumes (oracle/make_reference_checks.py)."""
    import make_reference_checks as mrc
    from r3g.vae import extract_near_surface_volume_fn
    z = _reference_checks(golden_dir)
    for n, x in mrc.nsm_inputs().items():
        for j, alpha in enumerate(mrc.NSM_ALPHAS):
            assert torch.equal(extract_near_surface_volume_fn(x.clone(), alpha), torch.from_numpy(z[f"nsm_{n}_{j}"]))


def test_flashvdm_resolution_schedule():
    """volume_decoders.py:310-320: 256 -> [63, 126, 252]; below min_resolution a single level."""
    from r3g.vae import FlashVDMVolumeDecoding
    dec = FlashVDMVolumeDecoding()
    with pytest.raises(ValueError):
        FlashVDMVolumeDecoding("nope")
    with pytest.raises(NotImplementedError):
        FlashVDMVolumeDecoding("merge")
    assert dec._topk(3072) == 1024 and dec._topk(512) == 256 and dec._topk(48) == 16
