"""CPU: the denoising step the flow-matching pipeline builds for its DiT (`_dit_step`), run eagerly on stub models --
which keyword arguments each kind of denoiser receives, that the step reads the buffers it returns, and that a model's
context k / v is projected once per call, not per step."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))


class _Plain:
    """A 2.0-style denoiser: forward(x, t, contexts, uncond_txt_shared=False)."""
    taps = None

    def __init__(self):
        self.calls = []

    def __call__(self, x, t, contexts, **kw):
        self.calls.append((x, t, contexts["main"], kw))
        return x + 1


class _Distilled(_Plain):
    guidance_embed = True


class _ContextKV(_Plain):
    """A 2mini-style denoiser whose cross-attention k / v of the context is projected by project_context."""

    def __init__(self):
        super().__init__()
        self.projections = 0

    def project_context(self, cond, out=None):
        self.projections += 1
        kv = cond.repeat(1, 1, 2)[None]
        if out is None:
            return kv
        return out.copy_(kv)


def _pipe(model):
    from r3g.pipelines import Hunyuan3DDiTFlowMatchingPipeline
    from r3g.scheduler import FlowMatchEulerDiscreteScheduler
    pipe = Hunyuan3DDiTFlowMatchingPipeline(vae=None, model=model, conditioner=None, image_processor=None,
                                            scheduler=FlowMatchEulerDiscreteScheduler(num_train_timesteps=1000),
                                            device="cpu")
    pipe.use_cuda_graph = False
    return pipe


@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("kind", ["plain", "distilled", "context_kv"])
def test_eager_step_passes_each_model_its_inputs(kind, shared):
    model = {"plain": _Plain, "distilled": _Distilled, "context_kv": _ContextKV}[kind]()
    pipe = _pipe(model)
    b = 1 if shared else 2
    x = torch.randn(b, 6, 4, dtype=torch.float16)
    ctx = torch.randn(b, 5, 3, dtype=torch.float16)
    x_in, t_buf, step = pipe._dit_step(x, ctx, shared, 5.0)
    assert x_in is x and t_buf.shape == (b,) and t_buf.dtype == torch.float16
    outs = [step() for _ in range(3)]
    assert len(model.calls) == 3 and pipe.replayed_launches == 0
    for (xs, ts, cs, kw), v in zip(model.calls, outs):
        assert xs is x_in and ts is t_buf and cs is ctx    # the loop updates these in place between steps
        assert torch.equal(v, x_in + 1)
        want = {"uncond_txt_shared"} | {"distilled": {"guidance"}, "context_kv": {"context_kv"}}.get(kind, set())
        assert set(kw) == want and kw["uncond_txt_shared"] is shared
        if kind == "distilled":
            assert kw["guidance"].dtype == torch.float16 and kw["guidance"].tolist() == [5.0] * b
        if kind == "context_kv":
            assert kw["context_kv"] is model.calls[0][3]["context_kv"]
            assert torch.equal(kw["context_kv"], ctx.repeat(1, 1, 2)[None])
    if kind == "context_kv":
        assert model.projections == 1
        pipe._dit_step(x, ctx, shared, 5.0)
        assert model.projections == 2      # once per call
