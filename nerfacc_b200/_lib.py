"""ctypes binding of ``csrc/libnerfacc_b200.so`` (the C ABI in ``include/nerfacc_b200.h``).

This module plays the role of the reference's ``nerfacc/cuda/__init__.py`` +
``_backend.py`` (lazy proxies around the pybind11 module): it is the only place
that touches the native library.  There is no CPU fallback and no JIT: if the
library is missing the import of any native entry point fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NFA_LIB") or os.path.join(_HERE, "csrc", "libnerfacc_b200.so")  # NFA_LIB: kernel-variant A/B runs

_c_i32, _c_i64, _c_f32, _c_ptr = C.c_int32, C.c_int64, C.c_float, C.c_void_p

# name -> (restype, argtypes).  Must list every symbol include/nerfacc_b200.h declares
# (tests/test_abi.py checks header == this table == the .so's exports).
SIGNATURES = {
    "nfa_version": (_c_i32, []),
    "nfa_error_string": (C.c_char_p, [_c_i32]),
    "nfa_ray_aabb_intersect": (_c_i32, [_c_i32, _c_ptr, _c_ptr, _c_i32, _c_ptr, _c_f32, _c_f32, _c_f32,
                                        _c_ptr, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_intersect_sorted": (_c_i32, [_c_i32, _c_ptr, _c_ptr, _c_i32, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_occ_words": (_c_i64, [_c_i32] * 4),
    "nfa_occ_coarse_words": (_c_i64, [_c_i32] * 4),
    "nfa_occ_pack": (_c_i32, [_c_i32] * 4 + [_c_ptr] * 5),
    "nfa_occ_ema_update": (_c_i32, [_c_i64, _c_ptr, _c_ptr, _c_f32, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_occ_threshold_workspace_bytes": (_c_i64, [_c_i64]),
    "nfa_occ_threshold_pack": (_c_i32, [_c_i32] * 4 + [_c_ptr, _c_f32] + [_c_ptr] * 6),
    "nfa_debug_set_march_trace": (None, [_c_ptr]),
    "nfa_march_workspace_bytes": (_c_i64, [_c_i32, _c_i64]),
    "nfa_march": (_c_i32, [_c_i32, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_f32, _c_f32, _c_i32, _c_i32, _c_i32, _c_i32,
                           _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_f32, _c_f32, _c_i64, _c_ptr,
                           _c_ptr, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_expand_samples": (_c_i32, [_c_i32, _c_i64, _c_ptr, _c_ptr, _c_f32, _c_f32, _c_i64, _c_ptr, _c_ptr, _c_ptr,
                                    _c_ptr, _c_ptr]),
    "nfa_expand_intervals": (_c_i32, [_c_i32, _c_i64, _c_ptr, _c_ptr, _c_f32, _c_i64, _c_i64] + [_c_ptr] * 10),
    "nfa_traverse_generic": (_c_i32, [_c_i32, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_i32, _c_i32, _c_i32, _c_i32,
                                      _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_f32, _c_f32, _c_i32, _c_i32]
                             + [_c_ptr] * 14),
    "nfa_counts_to_packed_info": (_c_i32, [_c_i32, _c_ptr, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_composite_fwd": (_c_i32, [_c_i32, _c_i64, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_i32, _c_ptr, _c_ptr, _c_ptr,
                                   _c_i32] + [_c_ptr] * 8),
    "nfa_composite_bwd": (_c_i32, [_c_i32, _c_i64, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_i32, _c_ptr, _c_ptr, _c_ptr,
                                   _c_i32] + [_c_ptr] * 10),
    "nfa_accumulate_fwd": (_c_i32, [_c_i32, _c_ptr, _c_ptr, _c_ptr, _c_i32, _c_ptr, _c_ptr]),
    "nfa_accumulate_atomic": (_c_i32, [_c_i64, _c_ptr, _c_ptr, _c_ptr, _c_i32, _c_ptr, _c_ptr]),
    "nfa_accumulate_bwd": (_c_i32, [_c_i64, _c_ptr, _c_ptr, _c_ptr, _c_i32, _c_ptr, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_scan_packed": (_c_i32, [_c_i32, _c_ptr, _c_ptr, _c_ptr, _c_i32, _c_i32, _c_i32, _c_i32, _c_ptr]),
    "nfa_scan_by_key_workspace_bytes": (_c_i64, [_c_i64]),
    "nfa_scan_by_key": (_c_i32, [_c_i64, _c_ptr, _c_ptr, _c_ptr, _c_i32, _c_i32, _c_i32, _c_ptr, _c_ptr]),
    "nfa_visibility_workspace_bytes": (_c_i64, [_c_i32, _c_i64]),
    "nfa_visibility_compact": (_c_i32, [_c_i32, _c_i64, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_i32, _c_f32, _c_f32]
                               + [_c_ptr] * 8),
    "nfa_vis_rounds_workspace_bytes": (_c_i64, [_c_i32, _c_i64]),
    "nfa_vis_rounds_begin": (_c_i32, [_c_i32, _c_i64, _c_ptr, _c_i32, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_vis_rounds_gather": (_c_i32, [_c_i32, _c_i64, _c_i32, _c_i32] + [_c_ptr] * 8),
    "nfa_vis_rounds_step": (_c_i32, [_c_i32, _c_i64, _c_i32, _c_i32, _c_i32, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_i32,
                                     _c_f32, _c_f32, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_vis_rounds_finish": (_c_i32, [_c_i32, _c_i64] + [_c_ptr] * 9),
    "nfa_render_test_workspace_bytes":(_c_i64, [_c_i32, _c_i32]),
    "nfa_render_test_begin": (_c_i32, [_c_i32, _c_i32, _c_f32, _c_ptr, _c_ptr]),
    "nfa_render_test_march": (_c_i32, [_c_i32, _c_i32, _c_i32, _c_ptr, _c_ptr, _c_f32, _c_i32, _c_i32, _c_i32, _c_i32]
                              + [_c_ptr] * 6 + [_c_f32, _c_f32, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_render_test_expand": (_c_i32, [_c_i32] * 5 + [_c_ptr] * 5),
    "nfa_render_test_composite": (_c_i32, [_c_i32] * 5 + [_c_i64] + [_c_ptr] * 5 + [_c_f32, _c_f32] + [_c_ptr] * 4),
    "nfa_render_test_finish": (_c_i32, [_c_i32, _c_i32] + [_c_ptr] * 7),
    "nfa_importance_sampling":(_c_i32, [_c_i32, _c_ptr, _c_ptr, _c_ptr, _c_i64, _c_i64, _c_ptr, _c_ptr, _c_i64, _c_i64,
                                         _c_i32, C.c_uint64, C.c_uint64] + [_c_ptr] * 8 + [_c_f32, _c_f32, _c_i32,
                                                                                          _c_ptr]),
    "nfa_searchsorted": (_c_i32, [_c_i64, _c_ptr, _c_ptr, _c_ptr, _c_i32, _c_i64, _c_ptr, _c_ptr, _c_i64, _c_ptr,
                                  _c_ptr, _c_ptr]),
    "nfa_pdf_loss_fwd": (_c_i32, [_c_i64, _c_i64, _c_ptr, _c_ptr, _c_i64, _c_ptr, _c_ptr, _c_f32, _c_ptr, _c_ptr]),
    "nfa_pdf_loss_bwd": (_c_i32, [_c_i64, _c_i64, _c_ptr, _c_ptr, _c_i64, _c_ptr, _c_ptr, _c_f32, _c_ptr, _c_ptr,
                                  _c_ptr]),
    "nfa_mailbox_create": (_c_i32, [_c_i32, _c_i32, _c_ptr, _c_ptr]),
    "nfa_mailbox_open": (_c_i32, [_c_ptr, _c_ptr]),
    "nfa_mailbox_close": (_c_i32, [_c_ptr]),
    "nfa_mailbox_destroy": (_c_i32, [_c_ptr]),
    "nfa_mailbox_post": (_c_i32, [_c_ptr, _c_ptr, _c_i32, _c_i32, _c_i32, C.c_uint32, _c_ptr]),
    "nfa_mailbox_sum": (_c_i32, [_c_ptr, _c_i32, _c_i32, C.c_uint32, _c_f32, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_pack_info_workspace_bytes": (_c_i64, [_c_i32]),
    "nfa_pack_info": (_c_i32, [_c_i64, _c_ptr, _c_i32, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_chunk_order_workspace_bytes": (_c_i64, []),
    "nfa_unpack_info": (_c_i32, [_c_i32, _c_ptr, _c_i64, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_unpack_rows": (_c_i32, [_c_i32, _c_ptr, _c_i64, _c_i64, _c_i64, _c_ptr, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_pack_rows": (_c_i32, [_c_i32, _c_ptr, _c_i64, _c_i64, _c_i64, _c_ptr, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_mask_counts": (_c_i32, [_c_i32, _c_i64, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_pack_masked": (_c_i32, [_c_i32, _c_i64, _c_i64, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_ptr]),
    "nfa_unpack_masked": (_c_i32, [_c_i32, _c_i64, _c_i64, _c_ptr, _c_ptr, _c_ptr, _c_ptr, _c_ptr]),
}

ABI_VERSION = 15
PDF_LOSS_MAX_INTERVALS = 16384  # NFA_PDF_LOSS_MAX_INTERVALS: nfa_pdf_loss_bwd's longest query row, in intervals

_lib = None
launches = 0  # number of native kernel-launching calls made through this module (bench.py reports it)


# Host work that may run while the host would otherwise wait for the GPU: the march has to finish before the
# batch size is known (the one sync of a sampling call), which leaves the host idle while the march runs.
# parallel.all_reduce_loss_async(defer=True) parks the NCCL enqueue of the previous step's loss here.
idle_tasks: list = []


def run_idle_tasks() -> None:
    while idle_tasks:
        idle_tasks.pop(0)()


def defer_until_wait(fn) -> None:
    """Run `fn()` the next time the library is about to wait for the GPU (inside the next sampling call,
    between queueing the march and waiting for its sample count).  Meant for host-side chores that need not
    happen now -- starting a copy of the next batch, a collective on last step's loss, a read-back for the
    logger -- on a step whose host side is the bottleneck."""
    idle_tasks.append(fn)


def load():
    """Load the shared library (once) and bind every entry point."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"nerfacc_b200: native library not found at {LIB_PATH}. Build it with "
            "`make -C nerfacc_b200/csrc` (or `python -c 'import __graft_entry__ as g; g.build()'`). "
            "There is no CPU or PyTorch fallback for the packed sampling/rendering path."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = header/library mismatch
        fn.restype = res
        fn.argtypes = args
    if lib.nfa_version() != ABI_VERSION:
        raise ImportError(f"nerfacc_b200: ABI version mismatch ({lib.nfa_version()} != {ABI_VERSION})")
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    """Map ABI return codes to the exception types the reference raises (TORCH_CHECK -> RuntimeError)."""
    if rc == 0:
        return
    msg = load().nfa_error_string(rc).decode()
    raise RuntimeError(f"nerfacc_b200.{what} failed: {msg} (code {rc})")


def ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


try:  # raw current-stream handle without building a torch.cuda.Stream object (~10x cheaper per launch)
    _raw_stream = torch._C._cuda_getCurrentRawStream
except AttributeError:  # pragma: no cover
    _raw_stream = None


def stream_ptr(device) -> int:
    if _raw_stream is not None:
        return _raw_stream(device.index if device.index is not None else torch.cuda.current_device())
    return torch.cuda.current_stream(device).cuda_stream


def require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        # reference: nerfacc/pack.py:47-48 (NotImplementedError), CHECK_CUDA in utils_cuda.cuh:12-17
        raise NotImplementedError(f"{what}: only CUDA tensors are supported for packed inputs.")


def call(name: str, device, *args) -> None:
    """Invoke a kernel-launching entry point on `device`'s current stream."""
    global launches
    fn = getattr(_lib if _lib is not None else load(), name)
    stream = stream_ptr(device)
    if device.index is None or device.index == torch.cuda.current_device():
        rc = fn(*args, stream)
    else:
        with torch.cuda.device(device):
            rc = fn(*args, stream)
    launches += 1
    if rc != 0:
        check(rc, name)
