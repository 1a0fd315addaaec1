"""FlowMatchEulerDiscreteScheduler and ConsistencyFlowMatchEulerDiscreteScheduler, interfaces of
Hunyuan3D-2/hy3dgen/shapegen/schedulers.py:55-318 and :325-480 (reversed-time Euler: sigmas run 0 -> 1).  Pure host
logic; the update itself is the fused r3g_cfg_euler_step kernel when the pipeline drives it, `step()` is kept for API
parity.  Both expose `step_sigmas()`, the sigma of every step plus the trailing 1.0: the pipeline steps from
step_sigmas()[i] to step_sigmas()[i + 1]."""
import types

import numpy as np
import torch


class FlowMatchEulerDiscreteSchedulerOutput:
    def __init__(self, prev_sample):
        self.prev_sample = prev_sample


class FlowMatchEulerDiscreteScheduler:
    order = 1

    def __init__(self, num_train_timesteps=1000, shift=1.0, use_dynamic_shifting=False):
        if use_dynamic_shifting:
            raise NotImplementedError("use_dynamic_shifting is not used by Hunyuan3D-2 shape checkpoints")
        self.config = types.SimpleNamespace(num_train_timesteps=num_train_timesteps, shift=shift,
                                            use_dynamic_shifting=False)
        t = torch.from_numpy(np.linspace(1, num_train_timesteps, num_train_timesteps, dtype=np.float32).copy())
        sig = t / num_train_timesteps
        sig = shift * sig / (1 + (shift - 1) * sig)
        self.timesteps = sig * num_train_timesteps
        self.sigmas = sig
        self.sigma_min, self.sigma_max = self.sigmas[-1].item(), self.sigmas[0].item()
        self._step_index = None
        self._begin_index = None
        self.num_inference_steps = None

    @property
    def step_index(self):
        return self._step_index

    def set_timesteps(self, num_inference_steps=None, device=None, sigmas=None, mu=None):
        """schedulers.py:181-221.  Kept on the HOST (the per-step scalars feed kernel arguments)."""
        n = self.config.num_train_timesteps
        if sigmas is None:
            self.num_inference_steps = num_inference_steps
            sigmas = np.linspace(self.sigma_max * n, self.sigma_min * n, num_inference_steps) / n
        sigmas = np.asarray(sigmas)
        sigmas = self.config.shift * sigmas / (1 + (self.config.shift - 1) * sigmas)
        s = torch.from_numpy(sigmas).to(dtype=torch.float32)
        self.timesteps = s * n
        self.sigmas = torch.cat([s, torch.ones(1)])
        self.num_inference_steps = len(self.timesteps)
        self._step_index = None

    def index_for_timestep(self, timestep):
        return _index_for_timestep(self.timesteps, timestep)

    def step_sigmas(self):
        return self.sigmas

    def output(self, step_index, sample, model_output, prev_sample):
        """What step() returns for the step from `sample` with `model_output` that produced `prev_sample`."""
        return FlowMatchEulerDiscreteSchedulerOutput(prev_sample)

    def step(self, model_output, timestep, sample, return_dict=True, **kwargs):
        """schedulers.py:245-318 on torch tensors (API parity; the pipeline uses the fused kernel instead)."""
        return _euler_step(self, model_output, timestep, sample, return_dict)

    def __len__(self):
        return self.config.num_train_timesteps


def _index_for_timestep(timesteps, timestep):
    """schedulers.py:223-236 / :414-426: the first step's index; with repeated timesteps, the second match."""
    idx = (timesteps == timestep).nonzero()
    return idx[1 if len(idx) > 1 else 0].item()


def _euler_step(sched, model_output, timestep, sample, return_dict):
    """schedulers.py:300-309 / :460-466: prev = fp32(sample) + (sigma_next - sigma) * model_output, in model_output's
    dtype; the sigmas are the scheduler's step_sigmas()."""
    if isinstance(timestep, int):
        raise ValueError("pass one of scheduler.timesteps, not an integer index")
    if sched._step_index is None:
        sched._step_index = sched.index_for_timestep(torch.as_tensor(timestep).cpu())
    i = sched._step_index
    sig = sched.step_sigmas()
    prev = (sample.to(torch.float32) + (sig[i + 1] - sig[i]).to(sample.device) * model_output).to(model_output.dtype)
    sched._step_index += 1
    return sched.output(i, sample, model_output, prev) if return_dict else (prev,)


class ConsistencyFlowMatchEulerDiscreteSchedulerOutput:
    def __init__(self, prev_sample, pred_original_sample):
        self.prev_sample = prev_sample
        self.pred_original_sample = pred_original_sample


class ConsistencyFlowMatchEulerDiscreteScheduler:
    """schedulers.py:330-480, the scheduler of the step-distilled `-turbo` checkpoints.  `sigmas` is the fixed
    pcm_timesteps table; set_timesteps picks `sigmas_`, the sigmas the steps actually use, from it."""
    order = 1

    def __init__(self, num_train_timesteps=1000, pcm_timesteps=50):
        self.config = types.SimpleNamespace(num_train_timesteps=num_train_timesteps, pcm_timesteps=pcm_timesteps)
        sigmas = np.linspace(0, 1, num_train_timesteps)
        step_ratio = num_train_timesteps // pcm_timesteps
        euler_timesteps = (np.arange(1, pcm_timesteps) * step_ratio).round().astype(np.int64) - 1
        self.euler_timesteps = np.asarray([0] + euler_timesteps.tolist())
        self.sigmas = torch.from_numpy(sigmas[self.euler_timesteps].copy()).to(dtype=torch.float32)
        self.timesteps = self.sigmas * num_train_timesteps
        self.sigmas_ = None
        self.num_inference_steps = None
        self._step_index = None
        self._begin_index = None

    @property
    def step_index(self):
        return self._step_index

    def set_timesteps(self, num_inference_steps=None, device=None, sigmas=None):
        """schedulers.py:382-412.  Of `sigmas` only the length is used: the pipeline's linspace(0, 1, N) asks for N
        steps, picked from the table at floor(linspace(0, pcm_timesteps, N, endpoint=False))."""
        n = num_inference_steps if num_inference_steps is not None else len(sigmas)
        if not 1 <= n <= self.config.pcm_timesteps:
            # more steps than table entries repeat a timestep; the reference then fails at its last step (IndexError)
            raise ValueError(f"ConsistencyFlowMatchEulerDiscreteScheduler: {n} inference steps, the schedule has "
                             f"pcm_timesteps = {self.config.pcm_timesteps} (1 <= steps <= pcm_timesteps)")
        self.num_inference_steps = n
        idx = np.floor(np.linspace(0, self.config.pcm_timesteps, num=n, endpoint=False)).astype(np.int64)
        s = self.sigmas[torch.from_numpy(idx)]
        self.timesteps = s * self.config.num_train_timesteps
        self.sigmas_ = torch.cat([s, torch.ones(1)])
        self._step_index = None
        self._begin_index = None

    def index_for_timestep(self, timestep):
        return _index_for_timestep(self.timesteps, timestep)

    def step_sigmas(self):
        return self.sigmas_

    def output(self, step_index, sample, model_output, prev_sample):
        """schedulers.py:468-477: pred_original_sample = fp32(sample) + (1 - sigma) * model_output, in its dtype."""
        sigma = self.sigmas_[step_index].to(sample.device)
        pred = (sample.to(torch.float32) + (1.0 - sigma) * model_output).to(model_output.dtype)
        return ConsistencyFlowMatchEulerDiscreteSchedulerOutput(prev_sample, pred)

    def step(self, model_output, timestep, sample, generator=None, return_dict=True):
        return _euler_step(self, model_output, timestep, sample, return_dict)

    def __len__(self):
        return self.config.num_train_timesteps
