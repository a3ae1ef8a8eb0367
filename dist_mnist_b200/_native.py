"""ctypes binding of the native runtime (`libdmnist_sm90a.so`, built in-tree by `_build.py`).

The C ABI is flat (see csrc/api.cu): kernel parameter blocks are ctypes mirrors of the structs in
csrc/protocol.h and are passed by address; `sizeof` of every mirror is checked against the library
at load time so a stale .so fails loudly instead of corrupting a launch.

On a box with a GPU the library is mandatory: `lib()` raises if it is missing (no silent fallback to
eager PyTorch for the hot ops). On a CPU-only box the same library provides the CPU plumbing backend
(POSIX shm + the native PS serve loop).
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import torch  # noqa: F401  (loads libcudart.so.12 that the native library links against)

from . import _build

MAX_WORKERS = 32

PUSH_LOCAL, PUSH_MAILBOX, PUSH_ATOMIC = 0, 1, 2
EPI_TRANSPOSED, EPI_ROWMAJOR_PUSH = 0, 1
LOSS_BOOK, LOSS_XENT = 0, 1
OPT_SGD, OPT_ADAM, OPT_MOMENTUM, OPT_ADAGRAD, OPT_RMSPROP = 0, 1, 2, 3, 4
OPT_ADADELTA, OPT_FTRL, OPT_PROXIMAL_ADAGRAD, OPT_PROXIMAL_SGD = 5, 6, 7, 8
APPLY_PER_PUSH, APPLY_MERGED = 0, 1
DT_F32, DT_BF16 = 0, 1
LR_CONSTANT, LR_EXPONENTIAL, LR_INVERSE_TIME, LR_NATURAL_EXP, LR_POLYNOMIAL, LR_COSINE, LR_PIECEWISE = range(7)
MAX_LR_BOUNDARIES = 8   # protocol.h kMaxLrBoundaries
CLIP_OFF, CLIP_GLOBAL_NORM, CLIP_NORM, CLIP_VALUE = range(4)   # protocol.h GradClipKind


class PushTarget(C.Structure):
    _fields_ = [
        ("mode", C.c_int),
        ("scale", C.c_float),
        ("base", C.c_void_p),
        ("slot_stride", C.c_uint64),
        ("flags", C.c_void_p),
        ("flag_slot_stride", C.c_uint32),
        ("nslots", C.c_uint32),
        ("gpu_scope", C.c_uint32),
        ("pad_", C.c_uint32),
        ("seq_ptr", C.c_void_p),
    ]


class GemmParams(C.Structure):
    _fields_ = [
        ("M", C.c_int), ("N", C.c_int), ("K", C.c_int),
        ("bn", C.c_int), ("stages", C.c_int), ("kc_per_split", C.c_int),
        ("epi", C.c_int), ("out_bf16", C.c_int), ("relu", C.c_int),
        ("ldo", C.c_int), ("ldmask", C.c_int), ("mask_bf16", C.c_int),
        ("out", C.c_void_p), ("bias", C.c_void_p), ("mask", C.c_void_p),
        ("colsum", PushTarget),
        ("colsum_offset", C.c_uint64),
        ("colsum_item_base", C.c_int), ("has_colsum", C.c_int),
        ("push", PushTarget),
        ("push_offset", C.c_uint64),
        ("push_item_base", C.c_int), ("push_staged", C.c_int),
        ("bump_seq", C.c_void_p),
        ("seq_counter", C.c_void_p),
        ("splitk_scratch", C.c_void_p),
        ("splitk_counter", C.c_void_p),
        ("debug_ts", C.c_void_p),
        ("splitk_cluster", C.c_int), ("pdl", C.c_int),
        ("pad2_", C.c_int), ("pad3_", C.c_int),
    ]


class StepResult(C.Structure):
    _fields_ = [("loss", C.c_float), ("global_step", C.c_uint32), ("correct", C.c_uint32), ("seq", C.c_uint32)]


class HeadParams(C.Structure):
    _fields_ = [
        ("B", C.c_int), ("B_pad", C.c_int), ("H", C.c_int), ("C", C.c_int),
        ("loss_kind", C.c_int), ("act_bf16", C.c_int), ("ldh", C.c_int), ("compute_grads", C.c_int),
        ("h", C.c_void_p), ("labels", C.c_void_p), ("w_last", C.c_void_p), ("b_last", C.c_void_p),
        ("dpre", C.c_void_p),
        ("push", PushTarget), ("push_bl", PushTarget), ("push_bh", PushTarget),
        ("off_w_last", C.c_uint64), ("off_b_last", C.c_uint64), ("off_b_hidden", C.c_uint64),
        ("item_w_last_base", C.c_int), ("item_b_last", C.c_int), ("item_b_hidden_base", C.c_int), ("pdl", C.c_int),
        ("result", C.c_void_p),
        ("seq_ptr", C.c_void_p), ("inbox", C.c_void_p), ("ps_global_step", C.c_void_p),
        ("nslots", C.c_uint32), ("n_inbox", C.c_uint32),
        ("debug_ts", C.c_void_p),
    ]


class PsItem(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("rows", C.c_int), ("cols", C.c_int), ("ld", C.c_int), ("flags", C.c_int),
                ("flag_index", C.c_int), ("pad_", C.c_int)]


class PsItemState(C.Structure):
    _fields_ = [("t", C.c_uint32), ("beta1_pow", C.c_float), ("beta2_pow", C.c_float), ("sched_step", C.c_uint32)]


class PsServeParams(C.Structure):
    _fields_ = [
        ("params", C.c_void_p), ("adam_m", C.c_void_p), ("adam_v", C.c_void_p), ("shadow_bf16", C.c_void_p),
        ("items", C.c_void_p), ("item_state", C.c_void_p),
        ("n_items", C.c_int), ("n_flags", C.c_int), ("n_workers", C.c_int), ("nslots", C.c_int), ("opt", C.c_int),
        ("apply_mode", C.c_int),
        ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float),
        ("mailbox", C.c_void_p), ("arena_elems", C.c_uint64),
        ("flags", C.c_void_p), ("next_seq", C.c_void_p), ("consumed", C.c_void_p),
        ("global_step", C.c_void_p), ("worker_done", C.c_void_p), ("host_stop", C.c_void_p),
        ("inbox_table", C.c_void_p),
        ("exit_counter", C.c_void_p),
        ("gpu_scope", C.c_uint32), ("lookahead", C.c_uint32),
        ("oneshot", C.c_uint32), ("ieee_math", C.c_uint32),
        ("stats", C.c_void_p),
        ("momentum", C.c_float), ("decay", C.c_float), ("nesterov", C.c_uint32), ("pad_", C.c_uint32),
        ("lr_schedule", C.c_int), ("decay_steps", C.c_uint32), ("decay_rate", C.c_float), ("end_lr", C.c_float),
        ("power", C.c_float), ("alpha", C.c_float), ("staircase", C.c_uint32), ("cycle", C.c_uint32),
        ("n_boundaries", C.c_int), ("boundaries", C.c_uint32 * MAX_LR_BOUNDARIES),
        ("values", C.c_float * (MAX_LR_BOUNDARIES + 1)),
        ("ema", C.c_void_p), ("ema_decay", C.c_float), ("ema_num_updates", C.c_uint32),
        ("l1", C.c_float), ("l2", C.c_float), ("l2_shrinkage", C.c_float), ("lr_power", C.c_float),
    ]


FUSED_CLUSTER = 8
FUSED_MAX_CHUNKS = 4
FUSED_MAX_SHARDS = 8
LANE_REC_WORDS = 16   # protocol.h kLaneRecWords
FUSED_ROW_TILE = 32   # rows of one row tile of the fused kernel; a batch occupies round_up(batch, 32) rows


class FusedSlice(C.Structure):
    _fields_ = [("kc_begin", C.c_int), ("kc_count", C.c_int), ("shard", C.c_int), ("flag_index", C.c_int),
                ("w_offset", C.c_uint64)]


class FusedShard(C.Structure):
    _fields_ = [("push", PushTarget), ("inbox", C.c_void_p)]


class FusedParams(C.Structure):
    _fields_ = [
        ("B", C.c_int), ("H", C.c_int), ("C", C.c_int), ("I", C.c_int),
        ("loss_kind", C.c_int), ("ldw", C.c_int), ("n_shards", C.c_int), ("strict", C.c_int),
        ("slice", FusedSlice * FUSED_CLUSTER),
        ("shard", FusedShard * FUSED_MAX_SHARDS),
        ("bias_h", C.c_void_p), ("w_last", C.c_void_p), ("b_last", C.c_void_p),
        ("shard_bh", C.c_int), ("shard_wl", C.c_int), ("shard_bl", C.c_int),
        ("flag_bh", C.c_int), ("flag_wl", C.c_int), ("flag_bl", C.c_int),
        ("off_bh", C.c_uint64), ("off_wl", C.c_uint64), ("off_bl", C.c_uint64),
        ("y_base", C.c_void_p),
        ("row_start", C.c_uint64), ("row_stride", C.c_uint64), ("row_wrap", C.c_uint64),
        ("n_steps", C.c_uint32), ("seq_base", C.c_uint32), ("nslots", C.c_uint32), ("stop_at", C.c_uint32),
        ("step_counter", C.c_void_p), ("stop_word", C.c_void_p), ("seq_word", C.c_void_p),
        ("ps_global_step", C.c_void_p),
        ("results", C.c_void_p),
        ("debug_ts", C.c_void_p),
        ("lane_rec", C.c_void_p),
        ("exit_counter", C.c_void_p),
        ("clear_stop", C.c_uint32), ("wait_acks", C.c_uint32),
        ("clip_kind", C.c_int), ("clip_norm", C.c_float), ("clip_min", C.c_float), ("clip_max", C.c_float),
        ("l2_scale", C.c_float), ("l2_biases", C.c_uint32),
    ]


GRAD_CLIP_MAX_VARS, GRAD_CLIP_MAX_SHARDS, GRAD_CLIP_BLOCKS = 8, 16, 132   # protocol.h kGradClip*


class GradClipVar(C.Structure):
    _fields_ = [("local", C.c_void_p), ("mailbox", C.c_void_p), ("mailbox_slot_stride", C.c_uint64),
                ("rows", C.c_uint32), ("cols", C.c_uint32), ("ld", C.c_uint32), ("pad_", C.c_uint32)]


class GradClipParams(C.Structure):
    _fields_ = [
        ("kind", C.c_int), ("clip_norm", C.c_float), ("clip_min", C.c_float), ("clip_max", C.c_float),
        ("n_vars", C.c_int), ("n_shards", C.c_int), ("nslots", C.c_uint32), ("gpu_scope", C.c_uint32),
        ("seq_ptr", C.c_void_p), ("partials", C.c_void_p),
        ("var", GradClipVar * GRAD_CLIP_MAX_VARS),
        ("flags", C.c_void_p * GRAD_CLIP_MAX_SHARDS),
        ("flag_slot_stride", C.c_uint32 * GRAD_CLIP_MAX_SHARDS),
        ("n_flags", C.c_uint32 * GRAD_CLIP_MAX_SHARDS),
        ("l2_w", C.c_void_p * GRAD_CLIP_MAX_VARS), ("l2_scale", C.c_float), ("l2_pad_", C.c_uint32),
        ("l2_partials", C.c_void_p), ("result", C.c_void_p),
    ]


class FusedMaps(C.Structure):
    _fields_ = [("w", (C.c_uint8 * 128) * FUSED_CLUSTER), ("xk", C.c_uint8 * 128),
                ("push", (C.c_uint8 * 128) * FUSED_CLUSTER)]


_MIRRORS = {
    "PushTarget": PushTarget, "GemmParams": GemmParams, "HeadParams": HeadParams, "StepResult": StepResult,
    "PsItem": PsItem, "PsItemState": PsItemState, "PsServeParams": PsServeParams,
    "FusedSlice": FusedSlice, "FusedShard": FusedShard, "FusedParams": FusedParams, "FusedMaps": FusedMaps,
    "GradClipVar": GradClipVar, "GradClipParams": GradClipParams,
}

WORKER_DEAD = 0xFFFFFFFF   # protocol.h kWorkerDead
TENSOR_MAP_BYTES = 128


class NativeError(RuntimeError):
    pass


_lib = None


def lib_path() -> Path:
    return _build.LIB_PATH


def _declare(l: C.CDLL) -> None:
    vp, i, u32, u64, sz, f = C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_size_t, C.c_float
    sigs = {
        "dm_last_error": (C.c_char_p, []),
        "dm_host_last_error": (C.c_char_p, []),
        "dm_sizeof": (i, [C.c_char_p]),
        "dm_device_count": (i, [C.POINTER(i)]),
        "dm_set_device": (i, [i]),
        "dm_device_sm_count": (i, [i, C.POINTER(i)]),
        "dm_device_cc": (i, [i, C.POINTER(i), C.POINTER(i)]),
        "dm_device_clock_khz": (i, [i, C.POINTER(i)]),
        "dm_cuda_malloc": (i, [i, sz, C.POINTER(vp)]),
        "dm_cuda_free": (i, [vp]),
        "dm_host_alloc": (i, [sz, C.POINTER(vp)]),
        "dm_host_free": (i, [vp]),
        "dm_ipc_get_handle": (i, [vp, vp]),
        "dm_ipc_open_handle": (i, [i, vp, C.POINTER(vp)]),
        "dm_ipc_close": (i, [vp]),
        "dm_can_access_peer": (i, [i, i, C.POINTER(i)]),
        "dm_enable_peer_access": (i, [i, i]),
        "dm_memcpy_async": (i, [vp, vp, sz, vp]),
        "dm_memset_async": (i, [vp, i, sz, vp]),
        "dm_stream_create": (i, [C.POINTER(vp)]),
        "dm_stream_destroy": (i, [vp]),
        "dm_stream_sync": (i, [vp]),
        "dm_stream_query": (i, [vp]),
        "dm_stream_wait_stream": (i, [vp, vp]),
        "dm_make_tensor_map_2d": (i, [vp, vp, i, u64, u64, u64, u32, u32]),
        "dm_make_tensor_map_3d": (i, [vp, vp, u64, u64, u64, u64, u64, u32, u32]),
        "dm_gemm_smem_bytes": (i, [i, i, i]),
        "dm_launch_gemm": (i, [vp, vp, vp, i, i, i, i, vp]),
        "dm_launch_head": (i, [vp, vp]),
        "dm_launch_accuracy": (i, [vp, vp, i, i, vp, vp]),
        "dm_launch_ps_serve": (i, [vp, i, i, vp]),
        "dm_launch_dense_apply": (i, [vp, vp, vp, vp, vp, sz, i, f, f, f, f, u32, vp]),
        "dm_launch_shadow_refresh": (i, [vp, vp, sz, vp]),
        "dm_launch_worker_done": (i, [vp, vp, vp]),
        "dm_launch_wait_ack": (i, [vp, u32, vp, vp]),
        "dm_launch_p2p_copy": (i, [vp, vp, sz, i, i, vp, u32, vp]),
        "dm_launch_p2p_reduce_apply": (i, [vp, vp, i, sz, f, i, vp]),
        "dm_launch_pingpong": (i, [vp, vp, i, i, vp, vp]),
        "dm_shm_create": (i, [C.c_char_p, sz, C.POINTER(vp)]),
        "dm_shm_open": (i, [C.c_char_p, sz, C.POINTER(vp)]),
        "dm_shm_unmap": (i, [vp, sz]),
        "dm_shm_unlink": (i, [C.c_char_p]),
        "dm_store_release_u32": (None, [vp, u32]),
        "dm_load_acquire_u32": (u32, [vp]),
        "dm_atomic_add_u32": (u32, [vp, u32]),
        "dm_wait_ge_u32": (i, [vp, u32, C.c_double]),
        "dm_cpu_ps_start": (vp, [vp]),
        "dm_cpu_ps_running": (i, [vp]),
        "dm_cpu_ps_applied": (u64, [vp]),
        "dm_cpu_ps_join": (i, [vp]),
        "dm_prepare_kernels": (i, [i]),
        "dm_exec_acquire_slot": (i, [vp, C.POINTER(i)]),
        "dm_exec_last_error": (C.c_char_p, []),
        "dm_loader_create": (vp, [vp, vp, sz, sz, sz, sz, sz, i, u64, i]),
        "dm_loader_next": (None, [vp, vp, vp]),
        "dm_loader_epochs": (u64, [vp]),
        "dm_loader_destroy": (None, [vp]),
        "dm_loader_enable_feed": (i, [vp, vp, vp, vp, vp, i]),
        "dm_loader_feed_enabled": (i, [vp]),
        "dm_copy_row_streaming": (None, [vp, vp, sz]),
        "dm_exec_create": (i, [i, i, i, i, sz, sz, C.POINTER(vp)]),
        "dm_exec_capture_stream": (vp, [vp, i]),
        "dm_exec_graph_steps": (i, [vp]),
        "dm_exec_begin_group_capture": (i, [vp, i]),
        "dm_exec_end_group_capture": (i, [vp, i]),
        "dm_exec_submit_group": (i, [vp, vp, vp, sz, vp, sz, C.POINTER(u64)]),
        "dm_exec_join": (i, [vp]),
        "dm_exec_fork": (i, [vp]),
        "dm_exec_slot_info": (i, [vp, i, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]),
        "dm_exec_compute_stream": (vp, [vp]),
        "dm_exec_copy_stream": (vp, [vp]),
        "dm_exec_nslots": (i, [vp]),
        "dm_exec_begin_capture": (i, [vp, i]),
        "dm_exec_end_capture": (i, [vp, i, i]),
        "dm_exec_submit": (i, [vp, vp, vp, C.POINTER(u64)]),
        "dm_exec_result": (i, [vp, u64, vp, i]),
        "dm_exec_drain": (i, [vp]),
        "dm_exec_run": (i, [vp, vp, u64, vp, u32, C.POINTER(u64)]),
        "dm_exec_run_resident": (i, [vp, u64, vp, vp, sz, sz, u64, u64, u64]),
        "dm_exec_submitted": (u64, [vp]),
        "dm_exec_kernel_launches": (u64, [vp]),
        "dm_exec_destroy": (i, [vp]),
        "dm_launch_fused": (i, [vp, vp, i, vp]),
        "dm_fused_max_lanes": (i, [i, i, C.POINTER(i)]),
        "dm_fused_max_lanes_clip": (i, [i, i, C.POINTER(i)]),
        "dm_fused_max_lanes_l2": (i, [i, i, i, C.POINTER(i)]),
        "dm_launch_grad_clip": (i, [C.c_void_p, i, C.c_void_p]),
        "dm_fused_smem_bytes": (i, [i]),
        "dm_nvls_probe": (i, [i, sz, i, C.c_char_p, sz]),
        "dm_fexec_last_error": (C.c_char_p, []),
        "dm_fexec_create": (i, [i, i, i, i, i, C.POINTER(vp)]),
        "dm_fexec_feed_stats": (None, [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]),
        "dm_fexec_buffers": (i, [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp),
                                 C.POINTER(i)]),
        "dm_fexec_set_params": (i, [vp, vp, vp]),
        "dm_fexec_compute_stream": (vp, [vp]),
        "dm_fexec_steps_done": (u64, [vp]),
        "dm_fexec_launches": (u64, [vp]),
        "dm_fexec_lanes": (i, [vp]),
        "dm_fexec_set_lanes": (i, [vp, i]),
        "dm_fexec_gather_threads": (i, [vp]),
        "dm_fexec_drain": (i, [vp]),
        "dm_fexec_debug": (i, [vp, vp]),
        "dm_fexec_steps_host": (i, [vp, vp, vp, u32, vp, C.POINTER(u32)]),
        "dm_fexec_run": (i, [vp, vp, u64, vp, u32, C.POINTER(u64), i]),
        "dm_fexec_run_resident": (i, [vp, vp, vp, u64, u64, u64, u64, i, i]),
        "dm_fexec_last_elapsed_ms": (i, [vp, C.POINTER(C.c_float)]),
        "dm_fexec_resident_results": (i, [vp, vp, u64, C.POINTER(u64)]),
        "dm_fexec_destroy": (i, [vp]),
    }
    for name, (res, args) in sigs.items():
        fn = getattr(l, name)
        fn.restype = res
        fn.argtypes = args


def lib(build_if_missing: bool = True) -> C.CDLL:
    """Load (building first if necessary) the native library. Raises NativeError if unavailable."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if os.environ.get("DM_NATIVE_LIB"):     # debugging aid: load an alternative build of the library (A/B runs)
        path = Path(os.environ["DM_NATIVE_LIB"])
        os.environ["DM_NO_BUILD"] = "1"
    if os.environ.get("DM_NO_BUILD") != "1":
        if not build_if_missing and not path.exists():
            raise NativeError(f"native library {path} is missing; run `python -m dist_mnist_b200._build`")
        try:
            if os.environ.get("DM_REBUILD") == "1":
                _build.build(force=True)
            else:
                _build.build_if_stale()   # content-hash check; no-op when the in-tree .so matches the sources
        except Exception as e:  # pragma: no cover - toolchain problems
            if not path.exists():
                raise NativeError(f"building {path} failed: {e}") from e
    try:
        l = C.CDLL(str(path))
    except OSError as e:
        raise NativeError(f"cannot load native library {path}: {e}") from e
    _declare(l)
    for name, cls in _MIRRORS.items():
        n = l.dm_sizeof(name.encode())
        if n != C.sizeof(cls):
            raise NativeError(
                f"ABI mismatch for {name}: library says {n} bytes, python mirror is {C.sizeof(cls)}; rebuild with "
                f"`python -m dist_mnist_b200._build --force`"
            )
    if l.dm_sizeof(b"CUtensorMap") != TENSOR_MAP_BYTES:
        raise NativeError("unexpected CUtensorMap size")
    _lib = l
    return l


def available() -> bool:
    try:
        lib()
        return True
    except NativeError:
        return False


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        l = lib()
        msg = (l.dm_last_error().decode() or l.dm_exec_last_error().decode() or l.dm_fexec_last_error().decode()
               or l.dm_host_last_error().decode())
        raise NativeError(f"{what or 'native call'} failed (rc={rc}): {msg}")


def current_stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


_prepared_devices = set()


def ensure_prepared(device: int | None = None) -> None:
    """Opt the big-shared-memory kernels in (cudaFuncSetAttribute) once per device, outside graph capture."""
    if device is None:
        device = torch.cuda.current_device()
    if device not in _prepared_devices:
        check(lib().dm_prepare_kernels(device), "prepare kernels")
        _prepared_devices.add(device)


def make_tensor_map_3d(ptr: int, dim0: int, dim1: int, dim2: int, stride1_bytes: int, stride2_bytes: int, box0: int,
                       box1: int):
    """3-D fp32 128-byte-swizzled tensor map [dim2][dim1][dim0], box {box0, box1, 1} (TMA-store destination)."""
    if stride1_bytes % 16 != 0 or stride2_bytes % 16 != 0:
        raise NativeError("TMA strides must be multiples of 16 bytes")
    buf = (C.c_uint8 * TENSOR_MAP_BYTES)()
    check(lib().dm_make_tensor_map_3d(C.addressof(buf), ptr, dim0, dim1, dim2, stride1_bytes, stride2_bytes, box0, box1),
          "cuTensorMapEncodeTiled(3d)")
    return buf


def make_tensor_map(ptr: int, dtype: int, dim0: int, dim1: int, stride1_bytes: int, box0: int, box1: int):
    """2-D 128-byte-swizzled (SWIZZLE_128B) tensor map over a row-major [dim1][dim0] tensor (dim0 contiguous).

    K-major and MN-major operand tiles use the same swizzle; the kernels address either layout themselves."""
    if stride1_bytes % 16 != 0:
        raise NativeError(f"TMA row stride must be a multiple of 16 bytes, got {stride1_bytes}")
    buf = (C.c_uint8 * TENSOR_MAP_BYTES)()
    check(
        lib().dm_make_tensor_map_2d(C.addressof(buf), ptr, dtype, dim0, dim1, stride1_bytes, box0, box1),
        "cuTensorMapEncodeTiled",
    )
    return buf


def nvls_probe(n_dev: int, nbytes: int, iters: int = 50) -> tuple[bool, str]:
    """NVSwitch multicast probe (csrc/nvls_sm90.cu): builds a multicast team over the first ``n_dev`` GPUs of this
    process, publishes ``nbytes`` from GPU 0 with ``multimem.st``, aggregates with ``multimem.ld_reduce`` and times both
    against unicast peer stores / loads. Returns ``(ok, log)``; never raises on a box without GPUs or NVLS."""
    buf = C.create_string_buffer(1 << 16)
    rc = lib().dm_nvls_probe(int(n_dev), int(nbytes), int(iters), buf, len(buf))
    return rc == 0, buf.value.decode(errors="replace")
