"""CPU: the machine code of the dual marching-cubes passes (cuobjdump on the in-tree libr3g.so): their output order comes
from the scans, so the emit kernels hold no global atomics, and none of the dual kernels spills."""
from test_sass import _one, sass  # noqa: F401  (module-scoped fixture)


def test_dual_emit_has_no_output_atomics(sass):  # noqa: F811
    funcs, _ = sass
    for needle in ("mc_dual_vertex_kernel", "mc_dual_face_kernel"):
        body = funcs[_one(funcs, needle)[0]]
        assert "ATOMG" not in body and "RED." not in body, needle + ": output order must come from the scans"


def test_dual_kernels_do_not_spill(sass):  # noqa: F811
    funcs, usage = sass
    for needle in ("mc_dual_vertex_kernel", "mc_dual_face_kernel"):
        name = _one(funcs, needle)[0]
        assert usage[name][1] == 0, f"{name}: {usage[name][1]} bytes of stack"
    # the dual eval pass keeps the Lewiner pass's frame: interior_joined takes the corner values through the stack
    name = _one(funcs, "mc_eval_kernelILb1E")[0]
    assert usage[name][1] == usage[_one(funcs, "mc_eval_kernelILb0E")[0]][1]
