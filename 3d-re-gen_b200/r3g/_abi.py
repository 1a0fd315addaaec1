"""ctypes binding of include/r3g.h.  This is the only place that touches the C ABI.

There is NO fallback: if libr3g.so is missing or no CUDA device is present, the first compute call
raises.  (`load_library()` itself works without a GPU so that the CPU test-suite can check the
exported symbols.)
"""
import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libr3g.so")

R3G_OK, R3G_E_INVALID, R3G_E_CUDA, R3G_E_WORKSPACE, R3G_E_LEVEL, R3G_E_NOSURFACE = 0, -1, -2, -3, -4, -5
R3G_MC_LEWINER, R3G_MC_DUAL = 0, 1
ATTN_MAX_WINDOWS = 2     # R3G_ATTN_MAX_WINDOWS


class LinearArgs(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("ldx", C.c_int64),
        ("w", C.c_void_p),
        ("bias", C.c_void_p),
        ("y", C.c_void_p), ("ldy", C.c_int64),
        ("M", C.c_int), ("N", C.c_int), ("K", C.c_int),
        ("seg_len", C.c_int), ("x_seg_stride", C.c_int64), ("y_seg_stride", C.c_int64),
        ("act", C.c_int), ("act_col0", C.c_int), ("act_col1", C.c_int),
        ("gate", C.c_void_p), ("gate_ld", C.c_int64), ("gate_rows", C.c_int),
        ("residual", C.c_void_p),
        ("out_f32", C.c_int),
        ("residual_f32", C.c_int),
        ("ls_gamma", C.c_void_p),
        ("qkn_mode", C.c_int), ("qkn_q_col0", C.c_int), ("qkn_k_col0", C.c_int), ("qkn_cols", C.c_int),
        ("qkn_eps", C.c_float),
        ("qkn_q_w", C.c_void_p), ("qkn_q_b", C.c_void_p), ("qkn_k_w", C.c_void_p), ("qkn_k_b", C.c_void_p),
        ("group_next", C.c_void_p),
        ("moe_mode", C.c_int), ("moe_groups", C.c_int), ("moe_experts", C.c_int), ("moe_top_k", C.c_int),
        ("moe_cap", C.c_int),
        ("moe_counts", C.c_void_p), ("moe_ids", C.c_void_p), ("moe_weights", C.c_void_p), ("moe_slots", C.c_void_p),
        ("moe_slot_x", C.c_void_p), ("moe_slot_scale", C.c_void_p), ("moe_slot_y", C.c_void_p),
    ]


class AttentionArgs(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("q_sb", C.c_int64), ("q_sh", C.c_int64), ("q_sl", C.c_int64),
        ("k", C.c_void_p), ("k_sb", C.c_int64), ("k_sh", C.c_int64), ("k_sl", C.c_int64),
        ("v", C.c_void_p), ("v_sb", C.c_int64), ("v_sh", C.c_int64), ("v_sl", C.c_int64),
        ("o", C.c_void_p), ("o_sb", C.c_int64), ("o_sh", C.c_int64), ("o_sl", C.c_int64),
        ("B", C.c_int), ("H", C.c_int), ("Lq", C.c_int), ("Lk", C.c_int),
        ("scale", C.c_float),
        ("win_row0", C.c_int * ATTN_MAX_WINDOWS), ("win_len", C.c_int * ATTN_MAX_WINDOWS),
        ("win_k0_count", C.c_int * ATTN_MAX_WINDOWS),
    ]


_vp, _i, _i64, _f, _sz = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_size_t

# name -> (restype, argtypes); mirrors include/r3g.h one to one (tests/test_abi.py checks the header against this)
SIGNATURES = {
    "r3g_version": (_i, []),
    "r3g_create": (_i, [_i, C.POINTER(_vp)]),
    "r3g_destroy": (None, [_vp]),
    "r3g_last_error": (C.c_char_p, [_vp]),
    "r3g_launch_count": (_i64, [_vp]),
    "r3g_mc_workspace_bytes": (_sz, [_i, _i, _i]),
    "r3g_mc_count": (_i, [_vp, _vp, _i, _i, _i, _f, _i, _vp, _sz, C.POINTER(_i64), C.POINTER(_i64), _vp]),
    "r3g_mc_extract": (_i, [_vp, _vp, _i, _i, _i, _f, _i, _vp, _vp, _sz, _vp, _vp, _vp]),
    "r3g_mc_classify": (_i, [_vp, _vp, _i, _i, _i, _f, _vp, _vp]),
    "r3g_mesh_components": (_i, [_vp, _vp, _i64, _i64, _vp, _vp]),
    "r3g_decimate_workspace_bytes": (_sz, [_i64, _i64]),
    "r3g_mesh_decimate": (_i, [_vp, _vp, _i64, _vp, _i64, _i64, _vp, _sz, _vp, _vp, C.POINTER(_i64), C.POINTER(_i64),
                               C.POINTER(_i64), _vp]),
    "r3g_linear": (_i, [_vp, C.POINTER(LinearArgs), _vp]),
    "r3g_attention": (_i, [_vp, C.POINTER(AttentionArgs), _vp]),
    "r3g_layernorm": (_i, [_vp, _vp, _i64, _vp, _i64, _i, _i, _f, _vp, _vp, _vp, _vp, _i64, _i, _i, _i64, _i64, _vp]),
    "r3g_layernorm_f32in": (_i, [_vp, _vp, _i64, _vp, _i64, _i, _i, _f, _vp, _vp, _vp]),
    "r3g_qk_norm_rope": (_i, [_vp, _vp, _i64, _i64, _i, _f, _vp, _vp, _vp, _vp, _f, _i, _i, _i, _vp]),
    "r3g_patchify": (_i, [_vp, _vp, _vp, _i64, _i, _i, _i, _i, _vp, _vp, _vp]),
    "r3g_qk_norm": (_i, [_vp, _vp, _i64, _i, _i, _i64, _i64, _i64, _i, _f, _vp, _vp, _vp, _vp, _i, _i64, _vp]),
    "r3g_gemv": (_i, [_vp, _vp, _vp, _vp, _i64, _vp, _i64, _vp, _i, _i, _i, _i, _i, _vp]),
    "r3g_swiglu": (_i, [_vp, _vp, _i64, _vp, _i64, _i64, _i, _vp]),
    "r3g_timestep_embedding": (_i, [_vp, _vp, _vp, _i, _i, _f, _f, _vp]),
    "r3g_cfg_euler_step": (_i, [_vp, _vp, _vp, _vp, _i64, _i, _f, _f, _vp]),
    "r3g_grid_fourier": (_i, [_vp, _vp, _i64, _i64, _i64, _i, _vp, _i, _i, _vp]),
    "r3g_points_fourier": (_i, [_vp, _vp, _vp, _i64, _i64, _i, _i, _vp]),
    "r3g_points_fourier_f32": (_i, [_vp, _vp, _vp, _i64, _i64, _i, _i, _vp]),
    "r3g_lnpost_dot": (_i, [_vp, _vp, _i64, _i, _i, _f, _vp, _vp, _vp, _vp, _vp, _vp]),
    "r3g_im2col3x3": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "r3g_bilinear_nhwc": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "r3g_gemv_f32": (_i, [_vp, _vp, _vp, _vp, _i64, _vp, _i64, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "r3g_layernorm_f32": (_i, [_vp, _vp, _i64, _vp, _i64, _i, _i, _f, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "r3g_small_attention_f32": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _f, _vp]),
    "r3g_unproject": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
}

_lib = None
_lock = threading.Lock()


class R3GError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"r3g error {code}: {msg}")
        self.code = code


def load_library():
    """dlopen libr3g.so and attach signatures.  Raises if the extension has not been built."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
                "r3g has no CPU fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
        return lib


class Context:
    """One r3g_ctx bound to one CUDA device."""

    def __init__(self, device=0):
        self.lib = load_library()
        self.handle = _vp()
        rc = self.lib.r3g_create(int(device), C.byref(self.handle))
        if rc != R3G_OK:
            msg = self.lib.r3g_last_error(self.handle).decode() if self.handle else "r3g_create failed"
            if self.handle:
                self.lib.r3g_destroy(self.handle)
                self.handle = None
            raise R3GError(rc, msg)
        self.device = int(device)

    def check(self, rc):
        if rc != R3G_OK:
            raise R3GError(rc, self.lib.r3g_last_error(self.handle).decode())

    @property
    def launches(self):
        return int(self.lib.r3g_launch_count(self.handle))

    def close(self):
        if getattr(self, "handle", None):
            self.lib.r3g_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_contexts = {}


def get_context(device=0):
    dev = int(device)
    ctx = _contexts.get(dev)
    if ctx is None:
        ctx = Context(dev)
        _contexts[dev] = ctx
    return ctx
