"""Build + ctypes binding of libbv2.so (C ABI in include/bv2.h).  No CPU fallback: importing works without
a GPU (so CPU-only hosts can inspect the ABI), but every compute entry point needs an sm_90 (H100) device."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(HERE, "libbv2.so")
SOURCES = [os.path.join(HERE, "csrc", "engine.cu")]
HEADERS = sorted(os.path.join(HERE, "csrc", f) for f in os.listdir(os.path.join(HERE, "csrc")) if f.endswith(".cuh")) + [
    os.path.join(ROOT, "include", "bv2.h")]
# kernel test harness (tests/cuda/kernel_harness.cu): the product headers behind an extern "C" test interface, same flags
HARNESS_SOURCE = os.path.join(ROOT, "tests", "cuda", "kernel_harness.cu")
HARNESS_PATH = os.path.join(HERE, "libbv2_kernel_harness.so")
# streaming harness (tests/cuda/stream_harness.cu): the Generator's window launches and wavefront planner, on top of the kernel harness
STREAM_HARNESS_SOURCE = os.path.join(ROOT, "tests", "cuda", "stream_harness.cu")
STREAM_HARNESS_PATH = os.path.join(HERE, "libbv2_stream_harness.so")
# bounded-stream harness (tests/cuda/stream_bounded_harness.cu): the resident-range planner and launches, on top of the kernel harness
BOUNDED_HARNESS_SOURCE = os.path.join(ROOT, "tests", "cuda", "stream_bounded_harness.cu")
BOUNDED_HARNESS_PATH = os.path.join(HERE, "libbv2_stream_bounded_harness.so")
# ragged-batch harness (tests/cuda/ragged_harness.cu): a k_g2_conv launch whose items stop at their own lengths, on top of the kernel harness
RAGGED_HARNESS_SOURCE = os.path.join(ROOT, "tests", "cuda", "ragged_harness.cu")
RAGGED_HARNESS_PATH = os.path.join(HERE, "libbv2_ragged_harness.so")
# ragged-stream harness (tests/cuda/ragged_stream_harness.cu): a k_g2_conv window of a ragged stream, on top of the bounded-stream harness
RAGGED_STREAM_HARNESS_SOURCE = os.path.join(ROOT, "tests", "cuda", "ragged_stream_harness.cu")
RAGGED_STREAM_HARNESS_PATH = os.path.join(HERE, "libbv2_ragged_stream_harness.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-shared"]

MAX_UPS, MAX_RK, MAX_DIL = 8, 4, 4


class Bv2Config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "n_vocab", "num_tones", "num_languages", "bert_dim", "inter_channels", "hidden_channels", "filter_channels",
        "n_heads", "n_layers", "kernel_size", "window_size", "gin_channels", "n_speakers", "n_flow_layer",
        "n_layers_trans_flow", "use_transformer_flow", "flow_kernel_size", "wn_layers", "upsample_initial_channel", "n_ups")] + [
        ("upsample_rates", C.c_int32 * MAX_UPS), ("upsample_kernel_sizes", C.c_int32 * MAX_UPS),
        ("n_resblock_kernels", C.c_int32), ("n_dilations", C.c_int32),
        ("resblock_kernel_sizes", C.c_int32 * MAX_RK), ("resblock_dilation_sizes", (C.c_int32 * MAX_DIL) * MAX_RK),
        ("sdp_filter", C.c_int32), ("sdp_kernel", C.c_int32), ("sdp_n_flows", C.c_int32), ("sdp_dds_layers", C.c_int32),
        ("sdp_num_bins", C.c_int32), ("sdp_tail_bound", C.c_float), ("dp_filter", C.c_int32), ("dp_kernel", C.c_int32),
        ("cond_layer_idx", C.c_int32), ("generator_precision", C.c_int32), ("n_flows", C.c_int32)]


#: every symbol include/bv2.h declares -> (restype, argtypes)
P, I64P, F32P = C.c_void_p, C.c_void_p, C.c_void_p
SYMBOLS = {
    "bv2_version": (C.c_char_p, []),
    "bv2_create": (C.c_int, [C.POINTER(P), C.POINTER(Bv2Config), C.c_int]),
    "bv2_create_sibling": (C.c_int, [C.POINTER(P), P]),
    "bv2_set_weight": (C.c_int, [P, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int, C.c_int]),
    "bv2_finalize": (C.c_int, [P]),
    "bv2_save_packed": (C.c_int, [P, C.c_char_p]),
    "bv2_load_packed": (C.c_int, [P, C.c_char_p]),
    "bv2_infer_begin": (C.c_int, [P, C.c_int, C.c_int, I64P, I64P, I64P, I64P, I64P, F32P, F32P, F32P, F32P, C.c_float,
                                  C.c_float, C.c_float, F32P, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "bv2_infer_begin_items": (C.c_int, [P, C.c_int, C.c_int, I64P, I64P, I64P, I64P, I64P, F32P, F32P, F32P, F32P, F32P, F32P, F32P,
                                        F32P, F32P, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "bv2_infer_begin_mix": (C.c_int, [P, C.c_int, C.c_int, I64P, I64P, C.c_int, I64P, F32P, I64P, I64P, F32P, F32P, F32P, F32P, F32P, F32P,
                                      F32P, F32P, F32P, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "bv2_infer_finish": (C.c_int, [P, F32P, C.c_int64, C.c_float, C.c_int32, F32P, F32P, F32P, F32P, F32P, F32P, F32P, C.c_void_p]),
    "bv2_infer_finish_pcm16": (C.c_int, [P, F32P, C.c_int64, C.c_float, C.c_int32, C.c_void_p, F32P, F32P, F32P, F32P, F32P, F32P, C.c_void_p]),
    "bv2_infer_finish_ragged": (C.c_int, [P, F32P, C.c_int64, C.c_float, C.c_int32, F32P, C.c_void_p, F32P, F32P, F32P, F32P, F32P, F32P,
                                          C.c_void_p]),
    "bv2_infer_finish_stream": (C.c_int, [P, F32P, C.c_int64, C.c_float, C.c_int32, F32P, F32P, F32P, F32P, F32P, F32P, F32P, C.c_void_p]),
    "bv2_stream_advance": (C.c_int, [P, C.c_int32, C.c_void_p, C.POINTER(C.c_int64)]),
    "bv2_infer_finish_stream_bounded": (C.c_int, [P, F32P, C.c_int64, C.c_float, C.c_int32, C.c_int32, F32P, F32P, F32P, F32P, F32P, F32P, F32P,
                                                  C.c_void_p]),
    "bv2_infer_finish_stream_ragged": (C.c_int, [P, F32P, C.c_int64, C.c_float, C.c_int32, C.c_int32, F32P, F32P, F32P, F32P, F32P, F32P, F32P,
                                                 C.c_void_p]),
    "bv2_stream_bytes": (C.c_int64, [P, C.c_int, C.c_int32, C.c_int32]),
    "bv2_wave_to_pcm16": (C.c_int, [P, C.c_int, C.c_int64, F32P, I64P, C.c_void_p, C.c_void_p]),
    "bv2_attn_path": (C.c_int, [P, F32P, C.c_void_p]),
    "bv2_reserve": (C.c_int, [P, C.c_int, C.c_int, C.c_int]),
    "bv2_reserve_stream": (C.c_int, [P, C.c_int, C.c_int, C.c_int, C.c_int32]),
    "bv2_text_encoder": (C.c_int, [P, C.c_int, C.c_int, I64P, I64P, I64P, I64P, I64P, F32P, F32P, F32P, F32P, F32P, F32P, C.c_void_p]),
    "bv2_duration": (C.c_int, [P, C.c_int, C.c_int, F32P, I64P, I64P, F32P, C.c_float, F32P, F32P, C.c_void_p]),
    "bv2_flow_reverse": (C.c_int, [P, C.c_int, C.c_int, F32P, I64P, I64P, F32P, C.c_void_p]),
    "bv2_generator": (C.c_int, [P, C.c_int, C.c_int, F32P, F32P, F32P, C.c_void_p]),
    "bv2_generator_ragged": (C.c_int, [P, C.c_int, C.c_int, F32P, F32P, I64P, F32P, C.c_void_p]),
    "bv2_debug_read": (C.c_int64, [P, C.c_char_p, C.c_void_p, C.c_int64]),
    "bv2_set_profiling": (C.c_int, [P, C.c_int]),
    "bv2_stage_ms": (C.c_float, [P, C.c_char_p]),
    "bv2_launch_count": (C.c_int64, [P]),
    "bv2_workspace_bytes": (C.c_int64, [P]),
    "bv2_workspace_grows": (C.c_int64, [P]),
    "bv2_peer_slab_alloc": (C.c_int, [C.c_int, C.c_int64, C.POINTER(C.c_void_p), C.c_void_p]),
    "bv2_peer_slab_open": (C.c_int, [C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]),
    "bv2_peer_slab_close": (C.c_int, [C.c_int, C.c_void_p]),
    "bv2_peer_slab_free": (C.c_int, [C.c_int, C.c_void_p]),
    "bv2_peer_write": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "bv2_last_error": (C.c_char_p, [P]),
    "bv2_destroy": (None, [P]),
}

_lock = threading.Lock()
_lib = None


def needs_build() -> bool:
    if not os.path.isfile(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(p) > t for p in SOURCES + HEADERS if os.path.isfile(p))


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile libbv2.so in-tree for sm_90a with nvcc (cross-compiles without a GPU)."""
    with _lock:
        if not force and not needs_build():
            return LIB_PATH
        tmp = LIB_PATH + ".tmp"  # link to a temporary name, then rename: a reader never sees a half-written library
        cmd = ["nvcc"] + NVCC_FLAGS + ["-o", tmp] + SOURCES
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
        os.replace(tmp, LIB_PATH)
        if verbose:
            print(r.stderr)
        return LIB_PATH


def _harness(stream: bool, bounded: bool, ragged: bool = False, ragged_stream: bool = False):
    """(source, library) of a test harness"""
    if ragged_stream:
        return RAGGED_STREAM_HARNESS_SOURCE, RAGGED_STREAM_HARNESS_PATH
    if ragged:
        return RAGGED_HARNESS_SOURCE, RAGGED_HARNESS_PATH
    if bounded:
        return BOUNDED_HARNESS_SOURCE, BOUNDED_HARNESS_PATH
    return (STREAM_HARNESS_SOURCE, STREAM_HARNESS_PATH) if stream else (HARNESS_SOURCE, HARNESS_PATH)


def harness_needs_build(stream: bool = False, bounded: bool = False, ragged: bool = False, ragged_stream: bool = False) -> bool:
    src, path = _harness(stream, bounded, ragged, ragged_stream)
    if not os.path.isfile(path):
        return True
    t = os.path.getmtime(path)
    deps = {HARNESS_SOURCE, src} | set(HEADERS) | ({BOUNDED_HARNESS_SOURCE} if ragged_stream else set())
    return any(os.path.getmtime(p) > t for p in deps if os.path.isfile(p))


def build_harness(force: bool = False, stream: bool = False, bounded: bool = False, ragged: bool = False, ragged_stream: bool = False) -> str:
    """Compile the kernel test harness (stream=True: the streaming harness, bounded=True: the bounded-stream harness, ragged=True:
    the ragged-batch harness, ragged_stream=True: the ragged-stream harness) next to libbv2.so with the product flags."""
    src, path = _harness(stream, bounded, ragged, ragged_stream)
    with _lock:
        if not force and not harness_needs_build(stream, bounded, ragged, ragged_stream):
            return path
        tmp = path + ".tmp"
        r = subprocess.run(["nvcc"] + NVCC_FLAGS + ["-o", tmp, src], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed ({os.path.basename(src)}):\n" + r.stdout + r.stderr)
        os.replace(tmp, path)
        return path


def load():
    """dlopen libbv2.so and type every exported symbol.  Raises if the library is missing (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} not built; run `python -c 'import __graft_entry__ as g; g.build()'`. "
                           "There is no CPU/PyTorch fallback for the engine.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
