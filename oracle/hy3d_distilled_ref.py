"""ORACLE -- test infrastructure only.  Nothing under 3d-re-gen_b200/ imports this file.

fp32 restatements of what a guidance-distilled Hunyuan3D-2 checkpoint (`hunyuan3d-dit-v2-0-fast` / `-turbo`) adds to
the base path restated in hy3d_ref.py: the guidance_in embedding of the DiT, the consistency scheduler's sigmas and
its step, and the denoise loop without classifier-free guidance.  Paths are relative to
Hunyuan3D-2/hy3dgen/shapegen/.  Pinned by tests/test_guidance_distilled.py against fixtures that
oracle/make_golden_distilled.py generated from the reference's own modules.
"""
import numpy as np
import torch
import torch.nn.functional as F

import hy3d_ref as R


def _uniform(n, stream):
    """n values in [-1, 1) from the splitmix64 finaliser of a counter: integer arithmetic only, so the same on every
    machine and library version."""
    z = (np.arange(n, dtype=np.uint64) + np.uint64(stream << 32)) * np.uint64(0x9E3779B97F4A7C15)
    z ^= z >> np.uint64(30)
    z *= np.uint64(0xBF58476D1CE4E5B9)
    z ^= z >> np.uint64(27)
    z *= np.uint64(0x94D049BB133111EB)
    z ^= z >> np.uint64(31)
    return (z >> np.uint64(40)).astype(np.float64) / 2.0 ** 23 - 1.0


def mini_state_dict(keys, shapes, seed):
    """The weights of a mini-geometry fixture, regenerated from its key names and shapes instead of being stored:
    linear weights U(-1, 1) / sqrt(fan_in) (the bound of nn.Linear's default init; x4 for guidance_in, so that its share
    of vec matters), biases 0.1 U, RMSNorm scales 1 + 0.25 U; every value rounded through fp16, as a GPU run holds it."""
    sd = {}
    for j, (k, shape) in enumerate(zip(keys, shapes)):
        k, shape = str(k), tuple(int(s) for s in shape if s > 0)      # shapes may be zero-padded to one width
        u = _uniform(int(np.prod(shape)), seed * 1000 + j).reshape(shape)
        if k.endswith("norm.scale"):
            v = 1 + 0.25 * u
        elif k.endswith(".bias"):
            v = 0.1 * u
        elif k.endswith(".weight") and len(shape) == 2:
            v = u / np.sqrt(shape[1]) * (4.0 if k.startswith("guidance_in.") else 1.0)
        else:
            raise ValueError(f"mini_state_dict: no rule for {k} {shape}")
        sd[k] = torch.from_numpy(v.astype(np.float16).astype(np.float32))
    return sd


def dit_forward(sd, x, t, cond, heads, depth, depth_single, guidance=None, taps=None):
    """Hunyuan3DDiT.forward, models/denoisers/hunyuan3ddit.py:381-410, with the guidance_embed branch of :392-396 when
    `guidance` is given.  The guidance embedding is taken in guidance's dtype (`1000 * guidance` in fp16 for the fp16
    pipeline's input) and then cast to the model's."""
    latent = R._lin(sd, "latent_in", x)
    temb = R.timestep_embedding(t, 256, max_period=1000.0, time_factor=1000.0).to(latent.dtype)
    vec = R._lin(sd, "time_in.out_layer", F.silu(R._lin(sd, "time_in.in_layer", temb)))
    if guidance is not None:
        gemb = R.timestep_embedding(guidance, 256, max_period=1000.0, time_factor=1000.0).to(latent.dtype)
        vec = vec + R._lin(sd, "guidance_in.out_layer", F.silu(R._lin(sd, "guidance_in.in_layer", gemb)))
    c = R._lin(sd, "cond_in", cond)
    for i in range(depth):
        latent, c = R.double_block(sd, f"double_blocks.{i}.", latent, c, vec, heads)
        if taps is not None:
            taps.append(torch.cat((c, latent), 1))
    latent = torch.cat((c, latent), 1)
    for i in range(depth_single):
        latent = R.single_block(sd, f"single_blocks.{i}.", latent, vec, heads)
        if taps is not None:
            taps.append(latent)
    latent = latent[:, c.shape[1]:]
    shift, scale = R._lin(sd, "final_layer.adaLN_modulation.1", F.silu(vec)).chunk(2, dim=1)
    latent = (1 + scale[:, None, :]) * R._ln(latent) + shift[:, None, :]
    return R._lin(sd, "final_layer.linear", latent)


def consistency_sigmas(num_inference_steps, pcm_timesteps, num_train_timesteps=1000):
    """schedulers.py:340-349 + :397-409: the pcm table, then the N entries at floor(linspace(0, pcm, N,
    endpoint=False)); returns (timesteps, sigmas_ with the trailing 1.0)."""
    table = np.linspace(0, 1, num_train_timesteps)
    ratio = num_train_timesteps // pcm_timesteps
    idx = np.asarray([0] + ((np.arange(1, pcm_timesteps) * ratio).round().astype(np.int64) - 1).tolist())
    table = torch.from_numpy(table[idx].copy()).to(torch.float32)
    pick = np.floor(np.linspace(0, pcm_timesteps, num=num_inference_steps, endpoint=False)).astype(np.int64)
    s = table[torch.from_numpy(pick)]
    return s * num_train_timesteps, torch.cat([s, torch.ones(1)])


def consistency_pred_original(sample, model_output, sigma):
    """schedulers.py:468-469."""
    return (sample.to(torch.float32) + (1.0 - sigma) * model_output).to(model_output.dtype)


def distilled_denoise_loop(sd, latents, cond, heads, depth, depth_single, steps, guidance_scale, pcm_timesteps,
                           t_dtype=None):
    """pipelines.py:708-759 for a guidance-distilled model: no CFG (batch B), the guidance scale as a model input
    ([guidance_scale] * B in the pipeline dtype fp16), the consistency scheduler's sigmas_.  t_dtype as in
    hy3d_ref.denoise_loop."""
    timesteps, sigmas = consistency_sigmas(steps, pcm_timesteps)
    guidance = torch.tensor([guidance_scale] * latents.shape[0], dtype=torch.float16).to(latents.device)
    for i, t in enumerate(timesteps):
        ts = t.expand(latents.shape[0]).to(t_dtype or latents.dtype) / 1000
        ts = ts.to(latents.dtype).to(latents.device)
        v = dit_forward(sd, latents, ts, cond, heads, depth, depth_single, guidance=guidance)
        latents = R.flow_euler_step(latents, v, sigmas[i], sigmas[i + 1])
    return latents
