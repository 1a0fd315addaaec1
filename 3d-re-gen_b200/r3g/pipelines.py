"""Shape-generation pipeline: interface of Hunyuan3D-2/hy3dgen/shapegen/pipelines.py
(Hunyuan3DDiTPipeline :135-677, Hunyuan3DDiTFlowMatchingPipeline :680-770, export_to_trimesh :94-109),
i.e. what src/2d_to_3d_models/run.py:77-84 calls:

    pipeline = Hunyuan3DDiTFlowMatchingPipeline.from_pretrained(path)            # or .from_random(...) here
    mesh = pipeline(image=img, num_inference_steps=50, octree_resolution=256, num_chunks=16000,
                    generator=torch.manual_seed(seed), output_type="trimesh")[0]

Everything between the conditioner output and the mesh runs in libr3g.so: 50 x (CFG-batched DiT forward +
fused CFG/Euler step), ShapeVAE transformer, dense SDF decode, marching cubes.
"""
import json
import os
import struct

import numpy as np
import torch

from . import ops
from .conditioner import DinoImageEncoder, SingleImageEncoder
from .dit import Hunyuan3DDiT
from .graphs import GraphCache
from .preprocessors import ImageProcessorV2
from .scheduler import FlowMatchEulerDiscreteScheduler, FlowMatchEulerDiscreteSchedulerOutput
from .vae import ShapeVAE, SurfaceExtractors

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
        network for checkpoints).  conditioner: "dinov2" (random-init DINOv2-giant through HF transformers) or
        None (callers then pass precomputed `cond=` tensors)."""
        cfg = config or HUNYUAN3D_2_CONFIG
        model = Hunyuan3DDiT(device=device, **cfg["model"]).init_random(seed)
        vae = ShapeVAE(device=device, **cfg["vae"]).init_random(seed + 1)
        sched = FlowMatchEulerDiscreteScheduler(**cfg["scheduler"])
        cond = None
        if conditioner == "dinov2":
            torch.manual_seed(seed + 2)
            cond = SingleImageEncoder(DinoImageEncoder(device=device, dtype=dtype, image_size=518))
        return cls(vae=vae, model=model, scheduler=sched, conditioner=cond,
                   image_processor=ImageProcessorV2(**cfg["image_processor"]), device=device, dtype=dtype, **kwargs)

    @classmethod
    def from_single_file(cls, ckpt_path, config_path, device="cuda", dtype=torch.float16, use_safetensors=None,
                         **kwargs):
        """pipelines.py:140-199: config.yaml with target/params entries + one checkpoint holding the `model`,
        `vae` and `conditioner` state dicts."""
        import yaml
        with open(config_path) as fh:
            config = yaml.safe_load(fh)
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
        model = Hunyuan3DDiT(device=device, **config["model"]["params"])
        model.load_state_dict(ckpt["model"])
        vae = ShapeVAE(device=device, **config["vae"]["params"])
        vae.load_state_dict(ckpt["vae"])
        # conditioner.py:239-246 + build_image_encoder: SingleImageEncoder(main_image_encoder={'type': ..., 'kwargs': ...})
        cc = config["conditioner"]
        if not str(cc.get("target", "")).endswith("SingleImageEncoder"):
            raise NotImplementedError(f"conditioner target {cc.get('target')!r}: only SingleImageEncoder (the "
                                      "Hunyuan3D-2 shape checkpoints' conditioner) is mirrored")
        enc_cfg = cc["params"]["main_image_encoder"]
        if enc_cfg.get("type") != "DinoImageEncoder":
            raise NotImplementedError(f"main_image_encoder type {enc_cfg.get('type')!r}: only DinoImageEncoder is mirrored")
        enc_kw = dict(enc_cfg.get("kwargs") or {})
        enc_kw.setdefault("image_size", 224)          # ImageEncoder.__init__ default (conditioner.py:62)
        enc = DinoImageEncoder(device=device, dtype=dtype, **enc_kw)
        if "conditioner" in ckpt:
            # conditioner.load_state_dict(ckpt['conditioner']) is strict in the reference (pipelines.py:179-180)
            pre = "main_image_encoder.model."
            bad = [k for k in ckpt["conditioner"] if not k.startswith(pre)]
            if bad:
                raise RuntimeError(f"unexpected conditioner keys (not under {pre!r}): {bad[:5]}")
            enc.model.load_state_dict({k[len(pre):]: v for k, v in ckpt["conditioner"].items()}, strict=True)
            enc.invalidate()
        return cls(vae=vae, model=model, scheduler=FlowMatchEulerDiscreteScheduler(**config["scheduler"]["params"]),
                   conditioner=SingleImageEncoder(enc),
                   image_processor=ImageProcessorV2(**config["image_processor"]["params"]), device=device,
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
                octree_resolution=256, mc_algo="mc", enable_pbar=True):
        if output_type == "latent":
            return latents
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        latents = (1.0 / self.vae.scale_factor * latents).contiguous()
        latents = self.vae(latents)
        ev[1].record()
        grid = self.vae.volume_decoder(latents, self.vae.geo_decoder, bounds=box_v, num_chunks=num_chunks,
                                       octree_resolution=octree_resolution, enable_pbar=enable_pbar)
        ev[2].record()
        outputs = self.vae.surface_extractor(grid, mc_level=mc_level, bounds=box_v,
                                             octree_resolution=octree_resolution)
        ev[3].record()
        torch.cuda.synchronize()
        self.timings.update(vae_ms=ev[0].elapsed_time(ev[1]), decode_ms=ev[1].elapsed_time(ev[2]),
                            mc_ms=ev[2].elapsed_time(ev[3]))
        self.last_grid = grid
        if output_type == "trimesh":
            outputs = export_to_trimesh(outputs)
        return outputs


class Hunyuan3DDiTFlowMatchingPipeline(Hunyuan3DDiTPipeline):

    def _denoise(self, latents, cond, timesteps, guidance_scale, callback=None, callback_steps=None):
        """pipelines.py:741-759.  Per step: DiT forward on cat([x, x]) with cat([cond, uncond]) (one CUDA graph
        replay), then the fused CFG mix + Euler update which also rewrites the duplicated model input."""
        B = latents.shape[0]
        n = len(timesteps)
        sig = self.scheduler.sigmas
        # timestep = t.expand(B).to(fp16) / num_train_timesteps, evaluated in fp16 as the reference does
        t16 = (timesteps.to(torch.float16) / self.scheduler.config.num_train_timesteps).to(self.device)
        # torch multiplies the fp16 model output by the 0-dim fp32 (sigma_next - sigma) after casting it to the
        # result dtype, fp16 (schedulers.py:305)
        dsig = [float((sig[i + 1] - sig[i]).to(torch.float16)) for i in range(n)]
        x = latents.contiguous()
        do_cfg = cond["main"].shape[0] == 2 * B
        x_in = torch.cat([x] * 2) if do_cfg else x
        t_buf = torch.full((x_in.shape[0],), 0.5, device=self.device, dtype=torch.float16)  # warm-up t; set per step
        ctx = {"main": cond["main"].contiguous()}
        g = None
        if self.use_cuda_graph and self.model.taps is None:
            g = self._graphs.get((x_in.shape, ctx["main"].shape), (x_in, t_buf, ctx["main"]),
                                 lambda xs, ts, cs: self.model(xs, ts, {"main": cs}))
            g.inputs[0].copy_(x_in)
            g.inputs[2].copy_(ctx["main"])
            x_in, t_buf = g.inputs[:2]
        for i in range(n):
            t_buf.copy_(t16[i].expand(x_in.shape[0]))
            if g is not None:
                g.replay()
                self.replayed_launches += g.launches
                v = g.outputs
            else:
                v = self.model(x_in, t_buf, ctx)
            if do_cfg:
                ops.cfg_euler_step_(x, v, guidance_scale, dsig[i], x_dup=x_in)
            else:
                ops.cfg_euler_step_(x, torch.cat([v, v]), 0.0, dsig[i], x_dup=None)
                x_in.copy_(x)
            if callback is not None and i % callback_steps == 0:
                # pipelines.py:757-759: callback(step_idx, t, outputs) with outputs.prev_sample = the new latents
                callback(i // getattr(self.scheduler, "order", 1), timesteps[i],
                         FlowMatchEulerDiscreteSchedulerOutput(prev_sample=x.clone()))   # x is updated in place
        return x

    @torch.inference_mode()
    def __call__(self, image=None, num_inference_steps=50, timesteps=None, sigmas=None, eta=0.0,
                 guidance_scale=5.0, generator=None, box_v=1.01, octree_resolution=384, mc_level=0.0, mc_algo=None,
                 num_chunks=8000, output_type="trimesh", enable_pbar=True, **kwargs):
        callback = kwargs.pop("callback", None)
        callback_steps = kwargs.pop("callback_steps", None)
        cond = kwargs.pop("cond", None)  # precomputed {'main': [2B, Lt, C]} skips the image encoder (bench/tests)
        latents = kwargs.pop("latents", None)
        self.set_surface_extractor(mc_algo)
        device, dtype = self.device, self.dtype
        do_cfg = guidance_scale >= 0
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
        latents = self._denoise(latents, cond, ts, guidance_scale, callback, callback_steps)
        ev[2].record()
        out = self._export(latents, output_type, box_v, mc_level, num_chunks, octree_resolution, mc_algo,
                           enable_pbar=enable_pbar)
        torch.cuda.synchronize()
        self.timings.update(cond_ms=ev[0].elapsed_time(ev[1]), denoise_ms=ev[1].elapsed_time(ev[2]))
        return out
