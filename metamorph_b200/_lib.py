"""ctypes binding of the C-ABI shared library (`metamorph_b200/_C.so`, see include/metamorph_b200.h).

The product path has NO fallback: if the library is missing, or an exported call fails, a
RuntimeError is raised (`MetaMorphB200Error`). PyTorch is used only for device memory + streams.
"""
from __future__ import annotations

import ctypes
from ctypes import c_char_p, c_float, c_int, c_longlong, c_void_p
from pathlib import Path

import torch

_SO = Path(__file__).resolve().parent / "_C.so"
_lib = None


class MetaMorphB200Error(RuntimeError):
    pass


def lib() -> ctypes.CDLL:
    """Load (once) and return the C-ABI library. Fails loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not _SO.exists():
            raise MetaMorphB200Error(
                f"{_SO} is missing: build it with `python -m metamorph_b200._build` "
                "(or __graft_entry__.build()). There is no CPU / eager fallback.")
        _lib = ctypes.CDLL(str(_SO))
        _lib.mm_last_error.restype = c_char_p
        _lib.mm_abi_version.restype = c_int
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().mm_last_error().decode(errors="replace")
        raise MetaMorphB200Error(f"{what} failed (code {rc}): {msg}")


def stream_ptr() -> c_void_p:
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t) -> c_void_p:
    if t is None:
        return c_void_p(0)
    return c_void_p(t.data_ptr())


def ll(x) -> c_longlong:
    return c_longlong(int(x))


# kernels launched per C-ABI call (for bench.py's `gpu_launches` claim); default 1
_LAUNCHES = {"mm_attn_bwd": 3, "mm_attn_bwd_tc": 2, "mm_attn_bwd_tc_varlen": 2, "mm_clip_coef": 1, "mm_decode_attn": 2,
             "mm_decode_attn_paged": 2, "mm_sumsq_bf16_accum": 2}
launch_count = 0


def call(name: str, *args) -> None:
    global launch_count
    fn = getattr(lib(), name)
    fn.restype = c_int
    check(fn(*args), name)
    launch_count += _LAUNCHES.get(name, 1)


def reset_launch_count() -> int:
    global launch_count
    n, launch_count = launch_count, 0
    return n


def require_cuda(*tensors) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise MetaMorphB200Error(
                "metamorph_b200 kernels run on CUDA (sm_90a) tensors only; got a CPU tensor. "
                "There is no CPU fallback on the product path.")


__all__ = ["lib", "call", "reset_launch_count", "check", "ptr", "ll", "stream_ptr", "require_cuda", "MetaMorphB200Error",
           "c_int", "c_float", "c_longlong", "c_void_p"]
