"""CPU: every ops.py wrapper reaches libr3g through ops._launch with the argument list of its C prototype, a tensor
argument must live on the launch's device, and a caller's out= buffer is checked before anything is launched.
_launch is replaced by a recorder that never calls the library, so nothing here touches a GPU."""
import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def ops():
    import __graft_entry__ as g
    g.build()                     # marching_cubes asks the library for r3g_mc_workspace_bytes
    from r3g import ops
    return ops


@pytest.fixture
def calls(ops, monkeypatch):
    """(entry point, arguments between the context and the stream) of every launch, tensors as their addresses."""
    rec = []

    def launch(name, anchor, *args):
        rec.append(("r3g_" + name, [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]))
    monkeypatch.setattr(ops, "_launch", launch)
    return rec


def h(*shape):
    return torch.zeros(shape, dtype=torch.float16)


def f(*shape):
    return torch.zeros(shape, dtype=torch.float32)


def _unproject(ops, out=None):
    E = np.tile(np.eye(4, dtype=np.float32)[:3], (2, 1, 1))
    K = np.tile(np.array([[8, 0, 3], [0, 8, 2], [0, 0, 1]], dtype=np.float32), (2, 1, 1))
    return ops.unproject(f(2, 4, 6) + 1, E, K, torch.float64, out=out)


# every public wrapper once, each allocating what it writes
VALID = [
    lambda ops: ops.linear(h(2, 4, 32), h(64, 32), h(64), act=ops.ACT_GELU_TANH, act_cols=(0, 32), gate=h(2, 64),
                           gate_rows=4, residual=h(2, 4, 64),
                           qk_norm=dict(mode=ops.QKN_LAYERNORM, q_col0=0, k_col0=None, cols=64, eps=1e-6, q_w=h(64),
                                        q_b=h(64))),
    lambda ops: ops.linear(h(4, 32), h(64, 32), None, out=f(4, 64), residual=f(4, 64), ls_gamma=f(64)),
    lambda ops: ops.linear_pair(dict(x=h(4, 32), w=h(64, 32)), dict(x=h(2, 32), w=h(64, 32), bias=h(64))),
    lambda ops: ops.attention(h(1, 8, 2, 64), h(1, 16, 2, 64), h(1, 16, 2, 64)),
    lambda ops: ops.layernorm(h(2, 4, 32), h(32), h(32), scale=h(2, 32), shift=h(2, 32), rows_per_batch=4),
    lambda ops: ops.layernorm_f32in(f(4, 32), h(32), h(32)),
    lambda ops: ops.qk_norm_rope_(h(4, 3 * 2 * 64), 2, 1e-5, h(64), h(64), h(64), h(64), 100.0, 4, 1, 3),
    lambda ops: ops.patchify(f(1, 3, 28, 28), 14, mean=(0.5, 0.5, 0.5), std=(0.2, 0.2, 0.2)),
    lambda ops: ops.qk_norm_(h(4, 3 * 128), 2, 0, 128, 64, 0, 1e-6, h(64), None, h(64), None),
    lambda ops: ops.gemv(h(16, 32), h(16), h(2, 32), silu_in=True),
    lambda ops: ops.swiglu(h(4, 64), 32),
    lambda ops: ops.timestep_embedding(h(2)),
    lambda ops: ops.cfg_euler_step_(h(1, 8, 4), h(2, 8, 4), 5.0, -0.02),
    lambda ops: ops.grid_fourier(h(27, 64), 0, 27, 2, [-1.0] * 3 + [1.0] * 3, 8, 0),
    lambda ops: ops.points_fourier(h(5, 3), h(5, 64), 8, 0),
    lambda ops: ops.points_fourier_f32(f(5, 3), h(5, 64), 8, 0),
    lambda ops: ops.lnpost_dot(h(5, 32), h(32), h(32), h(1, 32), h(1), f(5)),
    lambda ops: ops.im2col3x3(h(1, 4, 4, 8), stride=2),
    lambda ops: ops.bilinear_nhwc(h(1, 4, 4, 8), 7, 7),
    lambda ops: ops.gemv_f32(h(16, 32), f(16), f(2, 32), residual=f(2, 16), gamma=f(16)),
    lambda ops: ops.layernorm_f32(f(4, 32), shift=f(4, 32), scale=f(4, 32), gate=f(4, 32)),
    lambda ops: ops.small_attention_f32(f(2 * 5, 3 * 2 * 32), 2, 5, 2, 32),
    _unproject,
    lambda ops: ops.marching_cubes(f(5, 5, 5), 0.0, bounds=[-1.0] * 3 + [1.0] * 3),
    lambda ops: ops.mesh_components(torch.zeros(4, 3, dtype=torch.int32), 6),
    lambda ops: ops.mesh_decimate(f(6, 3), torch.zeros(4, 3, dtype=torch.int32), 2),
    lambda ops: ops.mc_classify(f(5, 5, 5)),
]

# wrapper -> (call with out=o, a correct out, {wrong kind: out the kernel must not be given})
OUTS = {
    "linear": (lambda ops, o: ops.linear(h(4, 32), h(64, 32), out=o), h(4, 64), {"dtype": torch.zeros(4, 64).char()}),
    "attention": (lambda ops, o: ops.attention(h(1, 8, 2, 64), h(1, 16, 2, 64), h(1, 16, 2, 64), out=o),
                  h(1, 8, 2, 64), {"shape": h(1, 8, 1, 64), "dtype": f(1, 8, 2, 64)}),
    "layernorm": (lambda ops, o: ops.layernorm(h(4, 32), out=o), h(4, 32), {"shape": h(4, 16), "dtype": f(4, 32)}),
    "layernorm_f32in": (lambda ops, o: ops.layernorm_f32in(f(4, 32), h(32), h(32), out=o), h(4, 32),
                        {"shape": h(3, 32), "dtype": f(4, 32), "layout": h(4, 64)[:, ::2]}),
    "gemv": (lambda ops, o: ops.gemv(h(16, 32), h(16), h(2, 32), out=o), h(2, 16),
             {"shape": h(2, 8), "dtype": f(2, 16), "layout": h(2, 32)[:, ::2]}),
    "swiglu": (lambda ops, o: ops.swiglu(h(4, 64), 32, out=o), h(4, 32),
               {"shape": h(4, 16), "dtype": f(4, 32), "layout": h(2, 4, 32)[:, :2]}),
    "timestep_embedding": (lambda ops, o: ops.timestep_embedding(h(2), out=o), h(2, 256),
                           {"shape": h(2, 128), "dtype": f(2, 256), "layout": h(256, 2).t()}),
    "cfg_euler_step_": (lambda ops, o: ops.cfg_euler_step_(h(1, 8, 4), h(2, 8, 4), 5.0, -0.02, x_dup=o), h(2, 8, 4),
                        {"shape": h(1, 8, 4), "dtype": f(2, 8, 4), "layout": h(2, 8, 8)[..., :4]}),
    "grid_fourier": (lambda ops, o: ops.grid_fourier(o, 0, 27, 2, [-1.0] * 3 + [1.0] * 3, 8, 0), h(27, 64),
                     {"shape": h(26, 64), "dtype": f(27, 64), "layout": h(27, 128)[:, :64]}),
    "points_fourier": (lambda ops, o: ops.points_fourier(h(5, 3), o, 8, 0), h(5, 64),
                       {"shape": h(4, 64), "dtype": f(5, 64)}),
    "points_fourier_f32": (lambda ops, o: ops.points_fourier_f32(f(5, 3), o, 8, 0), h(5, 64),
                           {"shape": h(4, 64), "dtype": f(5, 64)}),
    "lnpost_dot": (lambda ops, o: ops.lnpost_dot(h(5, 32), h(32), h(32), h(1, 32), h(1), o), f(5),
                   {"shape": f(4), "dtype": h(5), "layout": f(10)[::2]}),
    "im2col3x3": (lambda ops, o: ops.im2col3x3(h(1, 4, 4, 8), stride=2, out=o), h(4, 72),
                  {"shape": h(3, 72), "dtype": f(4, 72)}),
    "bilinear_nhwc": (lambda ops, o: ops.bilinear_nhwc(h(1, 4, 4, 8), 7, 7, out=o), h(1, 7, 7, 8),
                      {"shape": h(1, 6, 7, 8), "dtype": f(1, 7, 7, 8)}),
    "gemv_f32": (lambda ops, o: ops.gemv_f32(h(16, 32), f(16), f(2, 32), out=o), f(2, 16),
                 {"shape": f(2, 8), "dtype": h(2, 16)}),
    "layernorm_f32": (lambda ops, o: ops.layernorm_f32(f(4, 32), out=o), f(4, 32),
                      {"shape": f(3, 32), "dtype": h(4, 32)}),
    "small_attention_f32": (lambda ops, o: ops.small_attention_f32(f(10, 192), 2, 5, 2, 32, out=o), f(10, 64),
                            {"shape": f(10, 32), "dtype": h(10, 64)}),
    "unproject": (_unproject, f(2, 4, 6, 3).double(), {"shape": f(2, 4, 6, 2).double(), "dtype": f(2, 4, 6, 3)}),
}
BAD_OUTS = [pytest.param(op, kind, id=f"{op}-{kind}") for op, (_, _, bad) in OUTS.items() for kind in bad]


def test_argument_lists_match_the_c_signatures(ops, calls):
    from r3g import _abi
    for call in VALID:
        call(ops)
    for call, good, _ in OUTS.values():
        call(ops, good)
    compute = {name for name in _abi.SIGNATURES if name not in {
        "r3g_version", "r3g_create", "r3g_destroy", "r3g_last_error", "r3g_launch_count", "r3g_mc_workspace_bytes",
        "r3g_decimate_workspace_bytes"}}
    assert len(compute) == 26
    assert {name for name, _ in calls} == compute
    for name, args in calls:
        argtypes = _abi.SIGNATURES[name][1]
        assert len(args) == len(argtypes) - 2, name          # the context first and the stream last
        for i, (arg, argtype) in enumerate(zip(args, argtypes[1:-1]), 1):
            try:
                argtype.from_param(arg)
            except TypeError as e:
                pytest.fail(f"{name} argument {i} = {arg!r} does not convert to {argtype.__name__}: {e}")
    assert ops._PTR_ARGS["mesh_decimate"] == [0, 2, 5, 7, 8]


def test_tensor_arguments_must_live_on_the_launch_device(ops):
    with pytest.raises(ValueError, match="gemv: argument 3"):
        ops._ptr(torch.zeros(4), 0, "gemv", 3)
    assert ops._ptr(None, 0, "gemv", 2) is None
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops._launch("gemv", torch.zeros(4))


@pytest.mark.parametrize("op, kind", BAD_OUTS)
def test_a_wrong_out_is_refused_before_launch(ops, calls, op, kind):
    call, good, bad = OUTS[op]
    with pytest.raises(ValueError, match=op if kind != "layout" else None):
        call(ops, bad[kind])
    assert calls == []
    call(ops, good)
    assert len(calls) == 1
