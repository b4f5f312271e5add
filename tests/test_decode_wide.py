"""CPU tests of the 33..128-sequence decode path: the wide weight-streaming GEMM rejects bad arguments with
MetaMorphB200Error, and the decode engine / continuous batcher refuse more than 128 sequences, all before any device
work."""
from ctypes import c_int, c_void_p

import pytest
import torch


def _wide(x, w, m, epilogue=0, bias=c_void_p(0), resid=c_void_p(0), K=64, ld=64):
    from metamorph_b200._lib import call, ll
    call("mm_skinny_gemm_wide", x, w, c_void_p(256), bias, resid, ll(ld), ll(ld), ll(ld), ll(0), c_int(m), c_int(64),
         c_int(K), c_int(epilogue), c_int(0), c_void_p(0))


@pytest.fixture(scope="module", autouse=True)
def _built():
    from metamorph_b200 import _build
    _build.build(verbose=False)


def test_wide_gemm_rejects_bad_arguments_without_gpu():
    from metamorph_b200._lib import MetaMorphB200Error
    a = c_void_p(256)                                   # aligned, never dereferenced: every call fails its checks first
    for m in (0, 129, -1):
        with pytest.raises(MetaMorphB200Error, match=r"batch must be in \[1,128\]"):
            _wide(a, a, m)
    for epi in (-1, 5, 7):
        with pytest.raises(MetaMorphB200Error, match="bad epilogue"):
            _wide(a, a, 64, epilogue=epi)
    with pytest.raises(MetaMorphB200Error, match="16-byte aligned"):
        _wide(c_void_p(264), a, 64)
    with pytest.raises(MetaMorphB200Error, match="16-byte aligned"):
        _wide(a, c_void_p(258), 100)
    with pytest.raises(MetaMorphB200Error, match="K%32"):
        _wide(a, a, 40, K=48)
    with pytest.raises(MetaMorphB200Error, match="ldx/ldw"):
        _wide(a, a, 40, ld=60)
    with pytest.raises(MetaMorphB200Error, match="bias missing"):
        _wide(a, a, 40, epilogue=1)
    with pytest.raises(MetaMorphB200Error, match="residual missing"):
        _wide(a, a, 40, epilogue=2)


def test_more_than_128_sequences_are_refused_before_device_work():
    from metamorph_b200.engine.decode import DecodeEngine
    from metamorph_b200.engine.serve import ContinuousBatcher
    with pytest.raises(AssertionError, match="at most 128"):
        ContinuousBatcher(None, max_slots=129)
    with pytest.raises(AssertionError, match="at most 128"):
        ContinuousBatcher(None, max_slots=0)
    with pytest.raises(AssertionError, match="limited to 128"):
        DecodeEngine(None).generate(torch.zeros(129, 2, 8))
