"""Shape-generation pipeline: interface of Hunyuan3D-2/hy3dgen/shapegen/pipelines.py
(Hunyuan3DDiTPipeline :135-677, Hunyuan3DDiTFlowMatchingPipeline :680-770, export_to_trimesh :94-109),
i.e. what src/2d_to_3d_models/run.py:77-84 calls:

    pipeline = Hunyuan3DDiTFlowMatchingPipeline.from_pretrained(path)            # or .from_random(...) here
    mesh = pipeline(image=img, num_inference_steps=50, octree_resolution=256, num_chunks=16000,
                    generator=torch.manual_seed(seed), output_type="trimesh")[0]

Everything between the conditioner output and the mesh runs in libr3g.so: 50 x (CFG-batched DiT forward +
fused CFG/Euler step), ShapeVAE transformer, dense SDF decode, marching cubes.  A guidance-distilled checkpoint
(`hunyuan3d-dit-v2-0-fast` / `-turbo`: `guidance_embed: true`) runs without CFG, one sample per step with the guidance
scale as a model input; the `-turbo` config's ConsistencyFlowMatchEulerDiscreteScheduler gives its 5-step schedule.
A multi-view (Hunyuan3D-2mv) pipeline takes `image={'front': ..., 'left': ..., 'back': ..., 'right': ...}` (any
subset, any order): MVImageProcessorV2 stacks the views, DinoImageEncoderMV gives a V * 1370-row context, and the
same DiT runs on it.
"""
import json
import os
import struct

import numpy as np
import torch

from . import dist as r3g_dist
from . import ops
from .conditioner import DINOV2_LARGE, SingleImageEncoder, image_encoder_class
from .dit import Hunyuan3DDiT
from .dit_plain import HunYuanDiTPlain
from .graphs import GraphCache
from .preprocessors import ImageProcessorV2, MVImageProcessorV2
from .scheduler import ConsistencyFlowMatchEulerDiscreteScheduler, FlowMatchEulerDiscreteScheduler
from .vae import ShapeVAE, SurfaceExtractors, VanillaVolumeDecoder

# Hunyuan3D-2 `hunyuan3d-dit-v2-0/config.yaml` values.  The checkpoint config is downloaded at run time by the
# reference (utils.py:103-126) and is not in the source tree; these are the code defaults plus the published
# model card numbers (SURVEY.md section 8 preamble) and are constructor parameters everywhere.
HUNYUAN3D_2_CONFIG = dict(
    model=dict(in_channels=64, context_in_dim=1536, hidden_size=1024, mlp_ratio=4.0, num_heads=16, depth=16,
               depth_single_blocks=32, axes_dim=[64], theta=10000, qkv_bias=True, guidance_embed=False),
    vae=dict(num_latents=3072, embed_dim=64, num_freqs=8, include_pi=False, heads=16, width=1024,
             num_decoder_layers=16, qkv_bias=False, qk_norm=True, scale_factor=0.9990943042622529),
    scheduler=dict(num_train_timesteps=1000),
    image_processor=dict(size=512, border_ratio=0.15),
)

# The guidance- and step-distilled `hunyuan3d-dit-v2-0-turbo`: the same architecture plus guidance_in, stepped by
# ConsistencyFlowMatchEulerDiscreteScheduler.  pcm_timesteps = 100 is UNVERIFIED: the checkpoint's config.yaml is
# downloaded at run time and is not in the reference tree (the class default is 50).
HUNYUAN3D_2_TURBO_CONFIG = dict(
    HUNYUAN3D_2_CONFIG,
    model=dict(HUNYUAN3D_2_CONFIG["model"], guidance_embed=True),
    scheduler=dict(target="hy3dgen.shapegen.schedulers.ConsistencyFlowMatchEulerDiscreteScheduler",
                   num_train_timesteps=1000, pcm_timesteps=100),
)

# Hunyuan3D-2mv (`hunyuan3d-dit-v2-mv`, and `-mv-fast` / `-mv-turbo` below): up to four views of one object, each
# encoded by DINOv2 into 1370 tokens plus a per-view embedding, so the DiT's context holds V * 1370 rows.  The DiT and
# VAE are assumed to be 2.0's: UNVERIFIED, the checkpoints' config.yaml files are downloaded at run time and are not in
# the reference tree; the model zoo lists the same 1.1 B parameters and the reference pairs 2mv with the 2.0 VAE
# (pipelines.py:270,291).  view_num = 4 and image_size = 518 (1370 tokens per view) are likewise assumed.
HUNYUAN3D_2MV_CONFIG = dict(
    HUNYUAN3D_2_CONFIG,
    conditioner=dict(type="DinoImageEncoderMV", kwargs=dict(view_num=4, image_size=518, use_cls_token=True)),
    image_processor=dict(target="hy3dgen.shapegen.preprocessors.MVImageProcessorV2", size=512, border_ratio=0.15),
)

# `hunyuan3d-dit-v2-mv-turbo`: the multi-view conditioner with the -turbo DiT and scheduler (same UNVERIFIED
# assumptions as both configs above)
HUNYUAN3D_2MV_TURBO_CONFIG = dict(
    HUNYUAN3D_2_TURBO_CONFIG,
    conditioner=HUNYUAN3D_2MV_CONFIG["conditioner"],
    image_processor=HUNYUAN3D_2MV_CONFIG["image_processor"],
)

# Hunyuan3D-2mini (`hunyuan3d-dit-v2-mini`, 0.6 B parameters; the default of src/2d_to_3d_models/run.py:148,154): the
# HunYuanDiTPlain denoiser with a mixture-of-experts FFN in its last blocks, a 512-latent VAE and a DINOv2-large
# conditioner.  UNVERIFIED: the checkpoint's config.yaml is downloaded at run time and is not in the reference tree;
# every value below is an assumption, and every one is a constructor parameter.
HUNYUAN3D_2MINI_CONFIG = dict(
    model=dict(target="hy3dgen.shapegen.models.denoisers.hunyuandit.HunYuanDiTPlain", input_size=512, in_channels=64,
               hidden_size=1024, context_dim=1024, depth=16, num_heads=16, qk_norm=True, qk_norm_type="rms",
               text_len=1370, with_decoupled_ca=False, use_attention_pooling=False, qkv_bias=False,
               num_moe_layers=6, num_experts=8, moe_top_k=2),
    vae=dict(HUNYUAN3D_2_CONFIG["vae"], num_latents=512),
    scheduler=dict(num_train_timesteps=1000),
    conditioner=dict(type="DinoImageEncoder", kwargs=dict(config=DINOV2_LARGE, image_size=518, use_cls_token=True)),
    image_processor=dict(size=512, border_ratio=0.15),
)

# `hunyuan3d-dit-v2-mini-turbo`: HunYuanDiTPlain has no guidance embedding, so the turbo checkpoint is the same
# architecture run with CFG and the consistency scheduler (pcm_timesteps = 100 UNVERIFIED, as for 2.0-turbo)
HUNYUAN3D_2MINI_TURBO_CONFIG = dict(HUNYUAN3D_2MINI_CONFIG, scheduler=HUNYUAN3D_2_TURBO_CONFIG["scheduler"])

# `hunyuan3d-vae-v2-mini-withencoder` (minimal_vae_demo.py): ShapeVAE's constructor arguments, the 2mini VAE above plus
# the encoder's.  UNVERIFIED: the checkpoint's config.yaml is not in the reference tree; the encoder values are the
# constructor defaults of model.py:199-223 (5120 + 5120 surface points, as the demo's SharpEdgeSurfaceLoader samples).
HUNYUAN3D_2MINI_VAE_WITHENCODER_CONFIG = dict(
    HUNYUAN3D_2MINI_CONFIG["vae"], num_encoder_layers=8, pc_size=5120, pc_sharpedge_size=5120, point_feats=3,
    downsample_ratio=20, use_ln_post=True)


def denoiser_class(target):
    """The denoiser a config's `model.target` names (pipelines.py:121-128 instantiates it).  None: Hunyuan3DDiT, the
    2.0 / 2mv denoiser."""
    if target is None or str(target).endswith(".Hunyuan3DDiT"):
        return Hunyuan3DDiT
    if str(target).endswith(".HunYuanDiTPlain"):
        return HunYuanDiTPlain
    raise NotImplementedError(f"model target {target!r}: only Hunyuan3DDiT and HunYuanDiTPlain (the Hunyuan3D-2 / "
                              "-2mv / -2mini shape checkpoints') are mirrored")


def _context_kv(model):
    """A denoiser whose cross-attention k / v of the (step-invariant) context can be projected once per call
    (HunYuanDiTPlain.project_context): that method, else None."""
    return getattr(model, "project_context", None)


def _guidance_distilled(model):
    """pipelines.py:708-711 / :733-735: `hasattr(model, 'guidance_embed') and model.guidance_embed is True`."""
    return getattr(model, "guidance_embed", False) is True


def scheduler_class(target):
    """The scheduler a config's `scheduler.target` names (pipelines.py:184 instantiates it).  None: the flow-matching
    scheduler of the base checkpoints."""
    if target is None or str(target).endswith(".FlowMatchEulerDiscreteScheduler"):
        return FlowMatchEulerDiscreteScheduler
    if str(target).endswith(".ConsistencyFlowMatchEulerDiscreteScheduler"):
        return ConsistencyFlowMatchEulerDiscreteScheduler
    raise NotImplementedError(f"scheduler target {target!r}: only FlowMatchEulerDiscreteScheduler and "
                              "ConsistencyFlowMatchEulerDiscreteScheduler (the Hunyuan3D-2 shape checkpoints') are mirrored")


def image_processor_class(target):
    """The image processor a config's `image_processor.target` names (pipelines.py:182 instantiates it).  None: the
    single-view ImageProcessorV2."""
    name = None if target is None else str(target).rsplit(".", 1)[-1]
    if name is None or name == "ImageProcessorV2":
        return ImageProcessorV2
    if name == "MVImageProcessorV2":
        return MVImageProcessorV2
    raise NotImplementedError(f"image_processor target {target!r}: only ImageProcessorV2 and MVImageProcessorV2 (the "
                              "Hunyuan3D-2 / -2mv shape checkpoints') are mirrored")


class SimpleMesh:
    """Minimal stand-in for trimesh.Trimesh (trimesh is not installed in this image): vertices, faces, export()
    to .glb / .obj / .ply -- what src/2d_to_3d_models/run.py:99-102 needs from the returned object."""

    def __init__(self, vertices, faces):
        self.vertices = np.asarray(vertices, dtype=np.float32)
        self.faces = np.asarray(faces, dtype=np.int32)

    def export(self, path):
        ext = os.path.splitext(path)[1].lower()
        v, f = self.vertices, np.ascontiguousarray(self.faces.astype(np.uint32))
        if ext == ".obj":
            with open(path, "w") as fh:
                for p in v:
                    fh.write(f"v {p[0]:.8f} {p[1]:.8f} {p[2]:.8f}\n")
                for t in f + 1:
                    fh.write(f"f {t[0]} {t[1]} {t[2]}\n")
        elif ext == ".ply":
            with open(path, "wb") as fh:
                fh.write((f"ply\nformat binary_little_endian 1.0\nelement vertex {len(v)}\nproperty float x\n"
                          f"property float y\nproperty float z\nelement face {len(f)}\n"
                          "property list uchar int vertex_indices\nend_header\n").encode())
                fh.write(v.astype("<f4").tobytes())
                rec = np.empty(len(f), dtype=[("n", "u1"), ("i", "<i4", 3)])
                rec["n"], rec["i"] = 3, f
                fh.write(rec.tobytes())
        elif ext == ".glb":
            ib, vb = f.astype("<u4").tobytes(), v.astype("<f4").tobytes()
            doc = {"asset": {"version": "2.0", "generator": "r3g"}, "scene": 0, "scenes": [{"nodes": [0]}],
                   "nodes": [{"mesh": 0}],
                   "meshes": [{"primitives": [{"attributes": {"POSITION": 1}, "indices": 0, "mode": 4}]}],
                   "buffers": [{"byteLength": len(ib) + len(vb)}],
                   "bufferViews": [{"buffer": 0, "byteOffset": 0, "byteLength": len(ib), "target": 34963},
                                   {"buffer": 0, "byteOffset": len(ib), "byteLength": len(vb), "target": 34962}],
                   "accessors": [{"bufferView": 0, "componentType": 5125, "count": int(f.size), "type": "SCALAR"},
                                 {"bufferView": 1, "componentType": 5126, "count": len(v), "type": "VEC3",
                                  "min": v.min(0).tolist() if len(v) else [0, 0, 0],
                                  "max": v.max(0).tolist() if len(v) else [0, 0, 0]}]}
            js = json.dumps(doc, separators=(",", ":")).encode()
            js += b" " * (-len(js) % 4)
            bin_ = ib + vb
            bin_ += b"\0" * (-len(bin_) % 4)
            with open(path, "wb") as fh:
                fh.write(struct.pack("<4sII", b"glTF", 2, 12 + 8 + len(js) + 8 + len(bin_)))
                fh.write(struct.pack("<I4s", len(js), b"JSON") + js)
                fh.write(struct.pack("<I4s", len(bin_), b"BIN\0") + bin_)
        else:
            raise ValueError(f"unsupported mesh format {ext}")
        return path


def export_to_trimesh(mesh_output):
    """pipelines.py:94-109: reverse the face winding, wrap in a mesh object; None items stay None."""
    def one(m):
        if m is None:
            return None
        faces = m.mesh_f[:, ::-1]
        try:
            import trimesh
            return trimesh.Trimesh(m.mesh_v, faces)
        except ImportError:
            return SimpleMesh(m.mesh_v, faces)
    return [one(m) for m in mesh_output] if isinstance(mesh_output, list) else one(mesh_output)


def retrieve_timesteps(scheduler, num_inference_steps=None, device=None, timesteps=None, sigmas=None, **kwargs):
    """pipelines.py:37-91 (only the `sigmas=` form is used by the flow-matching pipeline)."""
    if timesteps is not None and sigmas is not None:
        raise ValueError("Only one of `timesteps` or `sigmas` can be passed.")
    if sigmas is not None:
        scheduler.set_timesteps(sigmas=sigmas, device=device, **kwargs)
    else:
        scheduler.set_timesteps(num_inference_steps, device=device, **kwargs)
    return scheduler.timesteps, len(scheduler.timesteps)


class Hunyuan3DDiTPipeline:
    def __init__(self, vae, model, scheduler, conditioner, image_processor, device="cuda", dtype=torch.float16,
                 **kwargs):
        self.vae, self.model, self.scheduler = vae, model, scheduler
        self.conditioner, self.image_processor = conditioner, image_processor
        self.device, self.dtype = torch.device(device), dtype
        self.kwargs = kwargs
        self.use_cuda_graph = True
        self._graphs = GraphCache(keep_all=True)
        self.replayed_launches = 0  # kernels executed through CUDA-graph replays (not seen by r3g_launch_count)
        self.timings = {}

    # -------------------------------------------------------------------------------- construction
    @classmethod
    def from_random(cls, seed=0, device="cuda", dtype=torch.float16, config=None, conditioner="dinov2",
                    **kwargs):
        """Architecture of tencent/Hunyuan3D-2 `hunyuan3d-dit-v2-0` with seeded random weights (there is no
        network for checkpoints).  conditioner: "dinov2" (random-init DINOv2-giant through HF transformers, of the
        config's `conditioner` type: DinoImageEncoder when it has none) or None (callers then pass precomputed `cond=`
        tensors).  The config's `image_processor.target` picks the image processor (image_processor_class)."""
        cfg = config or HUNYUAN3D_2_CONFIG
        mc = dict(cfg["model"])
        model = denoiser_class(mc.pop("target", None))(device=device, **mc).init_random(seed)
        vae = ShapeVAE(device=device, **cfg["vae"]).init_random(seed + 1)
        sc = dict(cfg["scheduler"])
        sched = scheduler_class(sc.pop("target", None))(**sc)
        cond = None
        if conditioner == "dinov2":
            enc = cfg.get("conditioner", dict(type="DinoImageEncoder", kwargs=dict(image_size=518)))
            torch.manual_seed(seed + 2)
            cond = SingleImageEncoder(image_encoder_class(enc["type"])(device=device, dtype=dtype, **enc["kwargs"]))
        ip = dict(cfg["image_processor"])
        return cls(vae=vae, model=model, scheduler=sched, conditioner=cond,
                   image_processor=image_processor_class(ip.pop("target", None))(**ip), device=device, dtype=dtype,
                   **kwargs)

    @classmethod
    def from_single_file(cls, ckpt_path, config_path, device="cuda", dtype=torch.float16, use_safetensors=None,
                         **kwargs):
        """pipelines.py:140-199: config.yaml with target/params entries + one checkpoint holding the `model`,
        `vae` and `conditioner` state dicts."""
        import yaml
        with open(config_path) as fh:
            config = yaml.safe_load(fh)
        sched_cls = scheduler_class(config["scheduler"].get("target"))
        proc_cls = image_processor_class(config["image_processor"].get("target"))
        if use_safetensors:
            ckpt_path = ckpt_path.replace(".ckpt", ".safetensors")
        if not os.path.exists(ckpt_path):
            raise FileNotFoundError(f"Model file {ckpt_path} not found")
        if use_safetensors:
            import safetensors.torch
            flat = safetensors.torch.load_file(ckpt_path, device="cpu")
            ckpt = {}
            for k, v in flat.items():
                name, rest = k.split(".", 1)
                ckpt.setdefault(name, {})[rest] = v
        else:
            ckpt = torch.load(ckpt_path, map_location="cpu", weights_only=True)
        model = denoiser_class(config["model"].get("target"))(device=device, **config["model"]["params"])
        model.load_state_dict(ckpt["model"])
        vae = ShapeVAE(device=device, **config["vae"]["params"])
        vae.load_state_dict(ckpt["vae"])
        # conditioner.py:239-246 + build_image_encoder: SingleImageEncoder(main_image_encoder={'type': ..., 'kwargs': ...})
        cc = config["conditioner"]
        if not str(cc.get("target", "")).endswith("SingleImageEncoder"):
            raise NotImplementedError(f"conditioner target {cc.get('target')!r}: only SingleImageEncoder (the "
                                      "Hunyuan3D-2 shape checkpoints' conditioner) is mirrored")
        enc_cfg = cc["params"]["main_image_encoder"]
        enc_cls = image_encoder_class(enc_cfg.get("type"))     # DinoImageEncoder, or DinoImageEncoderMV (2mv)
        enc_kw = dict(enc_cfg.get("kwargs") or {})
        enc_kw.setdefault("image_size", 224)          # ImageEncoder.__init__ default (conditioner.py:62)
        enc = enc_cls(device=device, dtype=dtype, **enc_kw)
        if "conditioner" in ckpt:
            # conditioner.load_state_dict(ckpt['conditioner']) is strict in the reference (pipelines.py:179-180); the
            # multi-view encoder's view_embed is a plain attribute there, not a state-dict entry
            pre = "main_image_encoder.model."
            bad = [k for k in ckpt["conditioner"] if not k.startswith(pre)]
            if bad:
                raise RuntimeError(f"unexpected conditioner keys (not under {pre!r}): {bad[:5]}")
            enc.model.load_state_dict({k[len(pre):]: v for k, v in ckpt["conditioner"].items()}, strict=True)
            enc.invalidate()
        return cls(vae=vae, model=model, scheduler=sched_cls(**config["scheduler"]["params"]),
                   conditioner=SingleImageEncoder(enc),
                   image_processor=proc_cls(**config["image_processor"]["params"]), device=device,
                   dtype=dtype, **kwargs)

    @classmethod
    def from_pretrained(cls, model_path, device="cuda", dtype=torch.float16, use_safetensors=True, variant="fp16",
                        subfolder="hunyuan3d-dit-v2-0", **kwargs):
        """pipelines.py:201-232 + utils.py:89-126: look under $HY3DGEN_MODELS (default ~/.cache/hy3dgen); the
        reference would fall back to a HuggingFace download, which needs a network this build does not have."""
        base = os.path.expanduser(os.path.join(os.environ.get("HY3DGEN_MODELS", "~/.cache/hy3dgen"), model_path,
                                               subfolder))
        if not os.path.isdir(base):
            raise FileNotFoundError(f"{base} not found and no network for snapshot_download; use "
                                    "Hunyuan3DDiTFlowMatchingPipeline.from_random() for synthetic weights")
        ext = "safetensors" if use_safetensors else "ckpt"
        vs = "" if variant is None else f".{variant}"
        return cls.from_single_file(os.path.join(base, f"model{vs}.{ext}"), os.path.join(base, "config.yaml"),
                                    device=device, dtype=dtype, use_safetensors=use_safetensors, **kwargs)

    def to(self, device=None, dtype=None):
        return self

    def compile(self):
        return None  # the reference torch.compile()s three modules; here the kernels are already native

    def enable_flashvdm(self, enabled=True, adaptive_kv_selection=True, topk_mode="mean", mc_algo="mc", replace_vae=True):
        """pipelines.py:258-290.  The reference also swaps in the `-turbo` VAE checkpoint when `replace_vae` and the
        model path is a known one; with no checkpoints reachable here the loaded VAE is kept."""
        self.vae.enable_flashvdm_decoder(enabled=enabled, adaptive_kv_selection=adaptive_kv_selection,
                                         topk_mode=topk_mode, mc_algo=mc_algo)

    def disable_flashvdm(self):
        self.vae.enable_flashvdm_decoder(False)

    # -------------------------------------------------------------------------------- pieces of __call__
    def set_surface_extractor(self, mc_algo):
        if mc_algo is None:
            return
        if mc_algo not in SurfaceExtractors:
            raise ValueError(f"Unknown mc_algo {mc_algo}")
        self.vae.surface_extractor = SurfaceExtractors[mc_algo]()

    def prepare_image(self, image):
        """pipelines.py:490-510: image (a path, PIL image or multi-view dict, or a list of them) -> {'image': the
        processors' tensors concatenated, 'mask': likewise, 'view_idxs': [one tuple per object] (multi-view only)}."""
        if isinstance(image, str) and not os.path.exists(image):
            raise FileNotFoundError(f"Couldn't find image at path {image}")
        images = image if isinstance(image, list) else [image]
        outs = [self.image_processor(im) for im in images]
        merged = {k: [o[k] for o in outs] for k in outs[0]}
        return {k: (torch.cat(v, 0) if isinstance(v[0], torch.Tensor) else v) for k, v in merged.items()}

    def encode_cond(self, image, additional_cond_inputs, do_classifier_free_guidance, dual_guidance=False):
        cond = self.conditioner(image=image, **additional_cond_inputs)
        if do_classifier_free_guidance:
            un = self.conditioner.unconditional_embedding(image.shape[0], **additional_cond_inputs)
            cond = {k: torch.cat([cond[k], un[k]], 0).to(self.dtype) for k in cond}
        return cond

    def prepare_latents(self, batch_size, dtype, device, generator, latents=None):
        """pipelines.py:473-488 with diffusers' randn_tensor: a CPU generator draws on the CPU in `dtype`."""
        shape = (batch_size, *self.vae.latent_shape)
        if latents is None:
            if generator is not None and generator.device.type == "cpu":
                latents = torch.randn(shape, generator=generator, device="cpu", dtype=dtype).to(device)
            else:
                latents = torch.randn(shape, generator=generator, device=device, dtype=dtype)
        else:
            latents = latents.to(device)
        return latents * getattr(self.scheduler, "init_noise_sigma", 1.0)

    def _export(self, latents, output_type="trimesh", box_v=1.01, mc_level=0.0, num_chunks=20000,
                octree_resolution=256, mc_algo="mc", enable_pbar=True, object_group=None):
        """VAE forward, volume decode, surface extraction.  With an object group of G > 1 members every member runs
        the VAE forward and decodes its balanced, contiguous share of the dense decode's query chunks; the leader
        receives the other shares into its grid and extracts the surface, the other members return [None].  FlashVDM's
        levels depend on the previous level's logits and are not split: with a group the leader runs the VAE forward,
        the decode and the extraction alone."""
        member, ranks = r3g_dist.group_layout(object_group)
        G = len(ranks)
        if output_type == "latent":
            return latents if member == 0 else [None]
        dec = self.vae.volume_decoder
        split = G > 1 and isinstance(dec, VanillaVolumeDecoder) and latents.shape[0] == 1
        self.timings.pop("gather_ms", None)
        if member != 0 and not split:       # nothing of this object's export runs here
            for k in ("vae_ms", "decode_ms", "mc_ms"):
                self.timings.pop(k, None)
            self.last_grid = None
            return [None]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        ev[0].record()
        latents = (1.0 / self.vae.scale_factor * latents).contiguous()
        latents = self.vae(latents)
        ev[1].record()
        kw = dict(bounds=box_v, num_chunks=num_chunks, octree_resolution=octree_resolution, enable_pbar=enable_pbar)
        if split:
            geo = self.vae.geo_decoder
            R = int(octree_resolution)
            ranges = r3g_dist.chunk_ranges(geo.grid_chunks(R)[1], G)
            grid = dec(latents, geo, chunks=ranges[member], **kw)
            ev[2].record()
            spans = [geo.chunk_span(R, c) for c in ranges]
            r3g_dist.gather_flat_slices(grid.view(-1), spans, object_group)
        else:
            grid = dec(latents, self.vae.geo_decoder, **kw)
            ev[2].record()
        ev[3].record()
        outputs = [None]
        if member == 0:
            outputs = self.vae.surface_extractor(grid, mc_level=mc_level, bounds=box_v,
                                                 octree_resolution=octree_resolution)
        ev[4].record()
        torch.cuda.synchronize()
        self.timings.update(vae_ms=ev[0].elapsed_time(ev[1]), decode_ms=ev[1].elapsed_time(ev[2]),
                            mc_ms=ev[3].elapsed_time(ev[4]))
        if split:
            self.timings.update(gather_ms=ev[2].elapsed_time(ev[3]))
        self.last_grid = grid
        if member != 0:
            return outputs
        if output_type == "trimesh":
            outputs = export_to_trimesh(outputs)
        return outputs


class Hunyuan3DDiTFlowMatchingPipeline(Hunyuan3DDiTPipeline):

    def _schedule(self, timesteps):
        """(t16, dsig) of `timesteps`.  t16: the model's timesteps, t.to(fp16) / num_train_timesteps evaluated in fp16
        as the reference does.  dsig[i]: sigma[i + 1] - sigma[i] rounded to fp16, because torch multiplies the fp16
        model output by the 0-dim fp32 (sigma_next - sigma) after casting it to the result dtype (schedulers.py:305)."""
        sig = self.scheduler.step_sigmas()
        t16 = (timesteps.to(torch.float16) / self.scheduler.config.num_train_timesteps).to(self.device)
        return t16, [float((sig[i + 1] - sig[i]).to(torch.float16)) for i in range(len(timesteps))]

    def _dit_step(self, x, ctx, shared, guidance_scale):
        """The DiT forward of one denoising step on the model input x [b, Li, C] and the context ctx [b, Lt, D].
        Returns (x_in, t_buf, step): the loop writes each step's timesteps into t_buf and may update x_in in place, and
        step() runs the forward on them and returns v.  With CUDA graphs on (and no taps to record), x_in and t_buf
        are static inputs of the graph for (x shape, ctx shape, shared), loaded with x, and step() is one replay.

        A guidance-distilled model also reads [guidance_scale] * b in fp16 (pipelines.py:733-737).  A model with
        project_context reads every block's cross-attention k / v of the context; they are the same at every step, so
        they are projected once per call, outside the step graph, into the buffer the step reads: a cached graph's
        static input, or else a new tensor that a capture copies into its own.  `shared` (the unconditional sample's
        text rows are all one vector, see Hunyuan3DDiT.forward's uncond_txt_shared) depends on this call's context, so
        the collapsed branch is chosen per call: `shared` is part of the graph key."""
        model, b = self.model, x.shape[0]
        t_buf = torch.full((b,), 0.5, device=self.device, dtype=torch.float16)  # warm-up t; set per step
        kw = {}
        if _guidance_distilled(model):
            kw["guidance"] = torch.tensor([guidance_scale] * b, dtype=torch.float16).to(self.device)
        graphed = self.use_cuda_graph and model.taps is None
        key = (x.shape, ctx.shape, shared)
        cached = self._graphs.entries.get(key) if graphed else None
        proj = _context_kv(model)
        if proj is not None:
            kw["context_kv"] = proj(ctx, out=None if cached is None else cached.inputs[-1])

        def forward(xs, ts, cs, *rest):
            return model(xs, ts, {"main": cs}, uncond_txt_shared=shared, **dict(zip(kw, rest)))

        inputs = (x, t_buf, ctx, *kw.values())
        if not graphed:
            return x, t_buf, lambda: forward(*inputs)
        g = self._graphs.get(key, inputs, forward)
        for dst, src in zip(g.inputs, inputs):
            if dst is not src:      # a cached graph's k / v were projected in place above
                dst.copy_(src)

        def replay():
            g.replay()
            self.replayed_launches += g.launches
            return g.outputs
        return g.inputs[0], g.inputs[1], replay

    def _denoise(self, latents, cond, timesteps, guidance_scale, callback=None, callback_steps=None):
        """pipelines.py:741-759.  Per step: one CUDA graph replay of the DiT forward, then the fused Euler update, which
        also rewrites the model input.  With CFG the forward runs on cat([x, x]) with cat([cond, uncond]) and the update
        mixes the two predictions first; without (a guidance-distilled model, or guidance_scale < 0) it runs on x."""
        B = latents.shape[0]
        t16, dsig = self._schedule(timesteps)
        x = latents.contiguous()
        ctx = cond["main"].contiguous()
        do_cfg = ctx.shape[0] == 2 * B
        # An unconditional context whose rows are all one vector (the zeros of unconditional_embedding) lets the DiT run
        # that sample on one text row (Hunyuan3DDiT.forward: uncond_txt_shared).  Checked once per call: one sync.
        shared = False
        if do_cfg and B == 1:
            un = ctx[1]
            shared = bool(torch.equal(un, un[:1].expand_as(un)))
        x_in, t_buf, step = self._dit_step(torch.cat([x] * 2) if do_cfg else x.clone(), ctx, shared, guidance_scale)
        for i in range(len(timesteps)):
            t_buf.copy_(t16[i].expand(x_in.shape[0]))
            v = step()
            report = callback is not None and i % callback_steps == 0
            x_prev = x.clone() if report else None
            ops.cfg_euler_step_(x, v, guidance_scale, dsig[i], x_dup=x_in)
            if report:
                # pipelines.py:757-759: callback(step_idx, t, outputs), outputs = what scheduler.step returns
                mixed = v
                if do_cfg:
                    vc, vu = v.chunk(2)
                    mixed = vu + guidance_scale * (vc - vu)
                callback(i // getattr(self.scheduler, "order", 1), timesteps[i],
                         self.scheduler.output(i, x_prev, mixed, x.clone()))   # x is updated in place
        return x

    def _denoise_group(self, latents, cond, timesteps, guidance_scale, group):
        """The denoising loop of one object on an object group.  With CFG, member 0 runs the conditional sample and
        member 1 the unconditional one (collapsed to one text row when its context allows, as in _denoise): each step
        is one graph replay of a B = 1 forward, the exchange of the two [Li, C] outputs into one (cond, uncond) buffer,
        and on both members the same fused CFG / Euler update as on one GPU, so x stays identical on both.  Without CFG
        member 0 denoises alone.  Members that hold no sample wait, then receive the final latents from the leader."""
        member, ranks = r3g_dist.group_layout(group)
        self.timings.pop("exchange_ms", None)
        B = latents.shape[0]
        if B != 1:
            raise ValueError(f"an object group generates one object per call, got a batch of {B}")
        n = len(timesteps)
        t16, dsig = self._schedule(timesteps)
        do_cfg = cond["main"].shape[0] == 2
        x = latents.contiguous().clone()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * n)]
        active = member < (2 if do_cfg else 1)
        if active:
            ctx = cond["main"][member:member + 1].contiguous()
            # the unconditional sample runs on one text row when all its rows are one vector (see _denoise)
            shared = bool(do_cfg and member == 1 and torch.equal(ctx[0], ctx[0, :1].expand_as(ctx[0])))
            # the Euler update below rewrites the model input in place: no copy per step
            x, t_buf, step = self._dit_step(x, ctx, shared, guidance_scale)
            v_pair = torch.empty((2,) + tuple(x.shape[1:]), device=self.device, dtype=x.dtype) if do_cfg else None
            for i in range(n):
                t_buf.copy_(t16[i].expand(1))
                v = step()
                if do_cfg:
                    ev[2 * i].record()
                    v = r3g_dist.exchange_cfg_pair(v, v_pair, group)
                    ev[2 * i + 1].record()
                ops.cfg_euler_step_(x, v, guidance_scale, dsig[i])
            x = x.clone()       # the graph's static input is rewritten by the next call
        r3g_dist.broadcast_from_leader(x, group, skip_pair=do_cfg)
        if active and do_cfg:
            torch.cuda.synchronize()
            self.timings["exchange_ms"] = sum(ev[2 * i].elapsed_time(ev[2 * i + 1]) for i in range(n))
        return x

    @torch.inference_mode()
    def __call__(self, image=None, num_inference_steps=50, timesteps=None, sigmas=None, eta=0.0,
                 guidance_scale=5.0, generator=None, box_v=1.01, octree_resolution=384, mc_level=0.0, mc_algo=None,
                 num_chunks=8000, output_type="trimesh", enable_pbar=True, **kwargs):
        callback = kwargs.pop("callback", None)
        callback_steps = kwargs.pop("callback_steps", None)
        cond = kwargs.pop("cond", None)  # precomputed {'main': [2B or B, Lt, C]} skips the image encoder (bench/tests)
        latents = kwargs.pop("latents", None)
        # a torch.distributed process group whose members generate this ONE object together (r3g/dist.py: object
        # groups); every member calls with the same arguments, the leader returns the output, the others [None]
        object_group = kwargs.pop("object_group", None)
        if object_group is not None and not r3g_dist.group_layout(object_group)[1][1:]:
            object_group = None     # a group of one is the single-GPU path
        self.set_surface_extractor(mc_algo)
        device, dtype = self.device, self.dtype
        # pipelines.py:708-711: a guidance-distilled model runs without CFG
        do_cfg = guidance_scale >= 0 and not _guidance_distilled(self.model)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        if cond is None:
            cond_inputs = self.prepare_image(image)
            image_t = cond_inputs.pop("image")
            if self.device.type == "cuda":       # the crop crosses PCIe once, from pinned memory, asynchronously
                image_t = image_t.pin_memory().to(self.device, non_blocking=True)
            cond = self.encode_cond(image_t, cond_inputs, do_cfg)
            batch_size = image_t.shape[0]
        else:
            batch_size = cond["main"].shape[0] // (2 if do_cfg else 1)
        ev[1].record()
        sigmas = np.linspace(0, 1, num_inference_steps) if sigmas is None else sigmas
        ts, num_inference_steps = retrieve_timesteps(self.scheduler, num_inference_steps, device, sigmas=sigmas)
        latents = self.prepare_latents(batch_size, dtype, device, generator, latents)
        if object_group is not None:
            if callback is not None:
                raise NotImplementedError("callback= is not supported with an object group")
            r3g_dist.check_same_inputs(object_group, latents, cond["main"])
            latents = self._denoise_group(latents, cond, ts, guidance_scale, object_group)
        else:
            latents = self._denoise(latents, cond, ts, guidance_scale, callback, callback_steps)
        ev[2].record()
        out = self._export(latents, output_type, box_v, mc_level, num_chunks, octree_resolution, mc_algo,
                           enable_pbar=enable_pbar, object_group=object_group)
        torch.cuda.synchronize()
        self.timings.update(cond_ms=ev[0].elapsed_time(ev[1]), denoise_ms=ev[1].elapsed_time(ev[2]))
        return out
