"""ctypes binding of libb2rl.so (the C ABI declared in include/b2rl.h).

There is deliberately no CPU fallback: if the shared library is missing the
GPU-backed classes raise ``B2rlLibraryError`` on first use.
"""
import ctypes
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(_HERE), "include")
LIB_PATH = os.path.join(CSRC, "libb2rl.so")
SOURCES = ["replay.cu", "sampler.cu", "step.cu", "gather.cu", "episodic.cu", "losses.cu", "ppo.cu", "sac.cu", "conv.cu", "gemm.cu"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3",
    "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
]


class B2rlLibraryError(RuntimeError):
    pass


class B2rlError(RuntimeError):
    def __init__(self, status, message):
        super().__init__("b2rl error %d: %s" % (status, message))
        self.status = status


def _sources():
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def build(force=False, verbose=False):
    """Compile libb2rl.so in-tree with nvcc for sm_90a (no GPU needed)."""
    srcs = _sources()
    deps = srcs + [os.path.join(CSRC, "b2rl_internal.cuh"), os.path.join(CSRC, "tree_dev.cuh"),
                   os.path.join(INCLUDE, "b2rl.h")]
    if (
        not force
        and os.path.exists(LIB_PATH)
        and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(d) for d in deps)
    ):
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-I", INCLUDE, "-o", LIB_PATH] + srcs
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd)
    return LIB_PATH


class ReplayConfig(ctypes.Structure):
    _fields_ = [
        ("capacity", ctypes.c_int64),
        ("part_capacity", ctypes.c_int64),
        ("part_bytes", ctypes.c_int32),
        ("stack", ctypes.c_int32),
        ("n_step", ctypes.c_int32),
        ("action_bytes", ctypes.c_int32),
        ("prioritized", ctypes.c_int32),
        ("device", ctypes.c_int32),
        ("max_batch", ctypes.c_int32),
        ("reserved", ctypes.c_int32),
    ]


class Experiences(ctypes.Structure):
    _fields_ = [
        ("state_parts", ctypes.c_void_p),
        ("next_parts", ctypes.c_void_p),
        ("action", ctypes.c_void_p),
        ("rewards", ctypes.c_void_p),
        ("len", ctypes.c_void_p),
        ("terminal", ctypes.c_void_p),
        ("priority", ctypes.c_void_p),
    ]


class BatchOut(ctypes.Structure):
    _fields_ = [
        ("state", ctypes.c_void_p),
        ("next_state", ctypes.c_void_p),
        ("action", ctypes.c_void_p),
        ("reward", ctypes.c_void_p),
        ("terminal", ctypes.c_void_p),
        ("discount", ctypes.c_void_p),
        ("step_rewards", ctypes.c_void_p),
        ("len", ctypes.c_void_p),
    ]


class StepArgs(ctypes.Structure):
    _fields_ = [
        ("n", ctypes.c_int32),
        ("mode", ctypes.c_int32),
        ("u", ctypes.c_void_p),
        ("u_on_device", ctypes.c_int32),
        ("norm", ctypes.c_int32),
        ("beta", ctypes.c_double),
        ("gamma_pow_host", ctypes.c_void_p),
        ("obs_mode", ctypes.c_int32),
        ("obs_scale", ctypes.c_float),
        ("index_dev", ctypes.c_void_p),
        ("priority_dev", ctypes.c_void_p),
        ("weight_dev", ctypes.c_void_p),
        ("prob_dev", ctypes.c_void_p),
        ("out", BatchOut),
    ]


SEQ_MAX_B, SEQ_MAX_LEAVES = 1024, 8


class SeqOut(ctypes.Structure):
    """b2rl_seq_out (include/b2rl.h)."""
    _fields_ = [("state", ctypes.c_void_p), ("next_state", ctypes.c_void_p),
                ("action", ctypes.c_void_p), ("reward", ctypes.c_void_p),
                ("terminal", ctypes.c_void_p)]


class SeqStates(ctypes.Structure):
    """b2rl_seq_states (include/b2rl.h)."""
    _fields_ = [("ring", ctypes.c_void_p), ("present", ctypes.c_void_p),
                ("ring_rows", ctypes.c_int64), ("row_floats", ctypes.c_int32),
                ("n_leaves", ctypes.c_int32),
                ("offset", ctypes.c_int32 * SEQ_MAX_LEAVES), ("d0", ctypes.c_int32 * SEQ_MAX_LEAVES),
                ("inner", ctypes.c_int32 * SEQ_MAX_LEAVES),
                ("out_state", ctypes.c_void_p * SEQ_MAX_LEAVES),
                ("out_next_state", ctypes.c_void_p * SEQ_MAX_LEAVES)]


class GemmOperand(ctypes.Structure):
    """b2rl_gemm_operand (include/b2rl.h)."""
    _fields_ = [("data", ctypes.c_void_p), ("mode", ctypes.c_int32), ("ld", ctypes.c_int32),
                ("row_off", ctypes.c_void_p), ("row_yx", ctypes.c_void_p),
                ("k_off", ctypes.c_void_p), ("k_yx", ctypes.c_void_p),
                ("y_limit", ctypes.c_int32), ("x_limit", ctypes.c_int32),
                ("lanes_along_k", ctypes.c_int32), ("u8", ctypes.c_int32),
                ("scale", ctypes.c_float)]


class GemmOutput(ctypes.Structure):
    """b2rl_gemm_output (include/b2rl.h)."""
    _fields_ = [("data", ctypes.c_void_p), ("ld", ctypes.c_int32),
                ("row_tab", ctypes.c_void_p), ("col_stride", ctypes.c_int32),
                ("bias", ctypes.c_void_p), ("relu", ctypes.c_int32)]


class TensorPair(ctypes.Structure):
    _fields_ = [("dst", ctypes.c_void_p), ("src", ctypes.c_void_p), ("numel", ctypes.c_int64)]


class PerInfo(ctypes.Structure):
    _fields_ = [
        ("total", ctypes.c_double),
        ("min", ctypes.c_double),
        ("max_priority", ctypes.c_double),
        ("napp", ctypes.c_int64),
        ("npop", ctypes.c_int64),
        ("scout_hits", ctypes.c_int32),
        ("reserved", ctypes.c_int32),
    ]


SAMPLE_EXACT, SAMPLE_PARALLEL = 0, 1
NORM_NONE, NORM_BATCH, NORM_MEMORY = 0, 1, 2
OBS_RAW, OBS_U8_TO_F32 = 0, 1

_vp, _i32, _i64, _dbl, _int = (
    ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_double, ctypes.c_int,
)

# name -> (restype, argtypes); lists every symbol of include/b2rl.h
SIGNATURES = {
    "b2rl_last_error": (ctypes.c_char_p, []),
    "b2rl_version": (ctypes.c_char_p, []),
    "b2rl_replay_create": (_int, [ctypes.POINTER(ReplayConfig), ctypes.POINTER(_vp)]),
    "b2rl_replay_destroy": (_int, [_vp]),
    "b2rl_replay_len": (_i64, [_vp]),
    "b2rl_replay_napp": (_i64, [_vp]),
    "b2rl_replay_npop": (_i64, [_vp]),
    "b2rl_replay_device_bytes": (_i64, [_vp]),
    "b2rl_replay_put_parts": (_int, [_vp, _vp, _int, _i64, _vp, _vp]),
    "b2rl_replay_append": (_int, [_vp, ctypes.POINTER(Experiences), _i64, _int, _vp]),
    "b2rl_per_sample": (_int, [_vp, _vp, _i32, _int, _vp, _vp, _vp]),
    "b2rl_per_weights": (_int, [_vp, _dbl, _int, _vp, _vp, _vp]),
    "b2rl_per_update_priorities": (_int, [_vp, _vp, _int, _i32, _vp]),
    "b2rl_per_update_errors": (_int, [_vp, _vp, _int, _i32, _dbl, _dbl, _dbl, _dbl, _vp]),
    "b2rl_per_get_info": (_int, [_vp, ctypes.POINTER(PerInfo), _vp]),
    "b2rl_per_read_priorities": (_int, [_vp, _i64, _i64, _vp, _vp]),
    "b2rl_per_read_tree": (_int, [_vp, _int, _i64, _i64, _vp, _vp]),
    "b2rl_per_set_max_priority": (_int, [_vp, _dbl, _vp]),
    "b2rl_replay_step": (_int, [_vp, ctypes.POINTER(StepArgs), _vp]),
    "b2rl_step_times": (_int, [_vp, _vp, _vp]),
    "b2rl_per_defer_errors": (_int, [_vp, _vp, _int, _i32, _dbl, _dbl, _dbl, _dbl]),
    "b2rl_host_priority_from_errors": (_int, [_vp, _i32, _dbl, _dbl, _int, _dbl, _int, _dbl, _vp]),
    "b2rl_per_update_host_errors": (_int, [_vp, _vp, _i32, _dbl, _dbl, _int, _dbl, _int, _dbl, _int, _vp]),
    "b2rl_per_flush": (_int, [_vp, _vp]),
    "b2rl_replay_gather": (
        _int, [_vp, _vp, _i32, _vp, _int, ctypes.c_float, ctypes.POINTER(BatchOut), _vp]),
    "b2rl_replay_gather_sequences": (
        _int, [_vp, _vp, _vp, _vp, _i32, _int, ctypes.c_float, ctypes.POINTER(SeqOut),
               ctypes.POINTER(SeqStates), _vp]),
    "b2rl_c51_loss_fwd": (_int, [_vp] * 7 + [_i32, _i32, _int] + [_vp] * 5),
    "b2rl_c51_loss_bwd": (_int, [_vp] * 4 + [_i32, _i32, _int, _vp, _vp]),
    "b2rl_td_loss_fwd": (_int, [_vp] * 7 + [_i32, _i32, _int, _int] + [_vp] * 6),
    "b2rl_td_loss_bwd": (_int, [_vp] * 5 + [_i32, _i32, _int, _int, _vp, _vp]),
    "b2rl_adv_td_loss_fwd": (_int, [_int] + [_vp] * 9 + [_i32, _i32, _dbl, _dbl, _int, _int]
                             + [_vp] * 6),
    "b2rl_quantile_huber_fwd": (_int, [_vp] * 4 + [_i32, _i32, _i32, _int] + [_vp] * 4),
    "b2rl_quantile_huber_bwd": (_int, [_vp] * 5 + [_i32, _i32, _i32, _int, _vp, _vp]),
    "b2rl_gae": (_int, [_vp] * 6 + [_i32, _i32, _dbl, _dbl] + [_vp] * 5),
    "b2rl_ppo_loss": (_int, [_vp] * 8 + [_i32, _dbl] + [ctypes.c_float] * 3 + [_vp] * 6),
    "b2rl_polyak": (_int, [ctypes.POINTER(TensorPair), _i32, _dbl, _vp]),
    "b2rl_sac_target": (_int, [_vp] * 7 + [ctypes.c_float, _i32, _vp, _vp]),
    "b2rl_conv_nature1_fwd": (_int, [_vp, _vp, _vp, _i32, _vp, _vp]),
    "b2rl_conv_nature1_fwd_u8": (_int, [_vp, ctypes.c_float, _vp, _vp, _i32, _vp, _vp]),
    "b2rl_gemm_workspace_bytes": (_i64, [_i32, _i32, _i32]),
    "b2rl_gemm_tf32x3": (_int, [_vp, _i32, _i32, _vp, _i32, _i32, _vp, _i32, _vp, _i32,
                                _i32, _i32, _i32, _vp, _i64, _vp]),
    "b2rl_gemm_debug_times": (_int, [_vp]),
    "b2rl_gemm_tf32x3_ex": (_int, [ctypes.POINTER(GemmOperand), ctypes.POINTER(GemmOperand),
                                   ctypes.POINTER(GemmOutput), _i32, _i32, _i32, _vp, _i64, _vp]),
}

_lib = None


def load():
    """Load libb2rl.so (built by ``build()`` / ``__graft_entry__.build()``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B2rlLibraryError(
            "%s not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). pfrl_b200 has no CPU fallback for its GPU classes." % LIB_PATH
        )
    L = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(L, name)  # AttributeError = header / library mismatch
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def check(status):
    if status != 0:
        raise B2rlError(status, load().b2rl_last_error().decode("utf-8", "replace"))
    return status
