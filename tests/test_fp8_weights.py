"""CPU tests of FP8 weights (DESIGN.md §1): the weight_dtype checks, FP8Weight's validation, the group view of the row
rule of oracle/kv_fp8.py on the rule's edge groups, and the argument refusals of the FP8 weight entry points."""
import numpy as np
import pytest
import torch

from oracle.kv_fp8 import E_MAX, NAN_BYTE, e4m3_decode, quantise_rows, row_exponent
from tests.test_kv_fp8 import _torch_bytes, edge_rows

BAD = ("fp8", "FP8_E4M3", "e4m3", "int8", None, torch.float8_e4m3fn, torch.bfloat16, 8, "")


def test_check_weight_dtype():
    from metamorph_b200.engine.decode import WEIGHT_DTYPES, check_weight_dtype
    assert WEIGHT_DTYPES == ("bf16", "fp8_e4m3")
    for ok in WEIGHT_DTYPES:
        check_weight_dtype(ok)
    for bad in BAD:
        with pytest.raises(ValueError, match="weight_dtype"):
            check_weight_dtype(bad)


class _NoDevice:
    """Stands in for the model: any attribute access is device work this test must not reach."""

    def __getattr__(self, name):
        raise AssertionError(f"touched model.{name} before refusing weight_dtype")


def test_bad_weight_dtype_is_refused_before_any_device_work():
    from metamorph_b200.engine.decode import DecodeEngine
    from metamorph_b200.engine.serve import ContinuousBatcher
    from metamorph_b200.model.metamorph_llama import MetaMorphLlamaForCausalLM
    emb = torch.zeros(1, 4, 256, dtype=torch.bfloat16)
    for bad in BAD:
        with pytest.raises(ValueError, match="weight_dtype"):
            DecodeEngine(_NoDevice()).generate(emb, max_new_tokens=2, weight_dtype=bad)
        stub = type("Stub", (), {})()
        stub._decode = DecodeEngine(_NoDevice())
        with pytest.raises(ValueError, match="weight_dtype"):
            MetaMorphLlamaForCausalLM.greedy_decode(stub, None, None, emb, max_new_tokens=2, weight_dtype=bad)
        with pytest.raises(ValueError, match="weight_dtype"):
            MetaMorphLlamaForCausalLM.generate(_NoDevice(), torch.zeros(1, 4, dtype=torch.long), weight_dtype=bad)
        with pytest.raises(ValueError, match="weight_dtype"):
            ContinuousBatcher(_NoDevice(), weight_dtype=bad)


def test_fp8_weight_validates_shapes_and_dtypes():
    from metamorph_b200.ops import FP8Weight
    q = torch.zeros(3, 256, dtype=torch.uint8)
    s = torch.ones(3, 2, dtype=torch.float32)
    w = FP8Weight(q, s)
    assert w.shape == (3, 256) and w.q is q and w.scale is s
    with pytest.raises(AttributeError):
        w.q = q
    bad = [
        (q.to(torch.int8), s, "uint8"),
        (q.view(torch.float8_e4m3fn), s, "uint8"),
        (q[None], s, "2-D"),
        (torch.zeros(3, 200, dtype=torch.uint8), s, "multiple of 128"),
        (torch.zeros(3, 0, dtype=torch.uint8), torch.ones(3, 0), "multiple of 128"),
        (q, s.double(), "scale"),
        (q, s.bfloat16(), "scale"),
        (q, torch.ones(3, 3), "scale"),
        (q, torch.ones(2, 2), "scale"),
        (q, torch.ones(6), "scale"),
        (torch.zeros(256, 3, dtype=torch.uint8).t(), s, "contiguous"),
        (q, torch.ones(2, 3).t(), "contiguous"),
    ]
    for qq, ss, msg in bad:
        with pytest.raises(ValueError, match=msg):
            FP8Weight(qq, ss)
    with pytest.raises(TypeError):
        FP8Weight(q.numpy(), s)


def edge_matrix():
    """W [N, 384] (three groups a row, an odd count) whose groups are the rule's edge rows, each in a different group
    slot, among random bf16 groups at spread-out scales."""
    rows = list(edge_rows().values())
    g = np.random.default_rng(11)
    N, ng = len(rows), 3
    w = g.standard_normal((N, ng, 128)) * np.ldexp(1.0, g.integers(-20, 20, (N, ng, 1)))
    w = torch.tensor(w).bfloat16().double().numpy()
    for i, r in enumerate(rows):
        w[i, i % ng] = r
    return w.reshape(N, ng * 128)


def test_group_view_of_the_row_rule_on_edge_groups():
    w = edge_matrix()
    N, K = w.shape
    q, sc, wh = quantise_rows(w.reshape(N, K // 128, 128))
    assert q.shape == (N, K // 128, 128) and sc.shape == (N, K // 128) and sc.dtype == np.float32
    for n in range(N):
        for j in range(K // 128):
            grp = w[n, 128 * j:128 * j + 128]
            if not np.all(np.isfinite(grp)):
                assert (q[n, j] == NAN_BYTE).all() and sc[n, j] == 1.0 and np.isnan(wh[n, j]).all()
                continue
            e = row_exponent(grp)
            assert sc[n, j] == 2.0 ** e
            assert np.array_equal(q[n, j], _torch_bytes(grp, e)), (n, j)
    # a group's bytes depend on that group alone: the same group quantised by itself
    one = quantise_rows(w[5, 128:256][None])
    assert np.array_equal(one[0][0], q[5, 1]) and one[1][0] == sc[5, 1]
    fin = np.isfinite(wh)
    assert np.array_equal(torch.tensor(wh[fin]).bfloat16().double().numpy(), wh[fin]), "W-hat is not a bf16 value"
    assert np.array_equal(wh, e4m3_decode(q) * sc[..., None].astype(np.float64), equal_nan=True)
    assert (sc == np.float32(2.0 ** E_MAX)).any(), "no group at e = 120"


def test_fp8_weight_entry_points_refuse_bad_arguments_without_gpu():
    from ctypes import c_int, c_void_p
    from metamorph_b200._lib import MetaMorphB200Error, call, ll
    n, a = c_void_p(0), c_void_p(256)
    gemm_args = lambda K, ldw, lds, sc, m=4: (a, a, sc, a, n, n, ll(K), ll(ldw), ll(lds), ll(64), ll(0), c_int(m),  # noqa: E731
                                               c_int(64), c_int(K), c_int(0), c_int(0), n)
    for name, mmax in (("mm_skinny_gemm_fp8", 32), ("mm_skinny_gemm_wide_fp8", 128)):
        with pytest.raises(MetaMorphB200Error, match="batch"):
            call(name, *gemm_args(256, 256, 2, a, m=mmax + 1))
        with pytest.raises(MetaMorphB200Error, match="K%128"):
            call(name, *gemm_args(192, 192, 2, a))
        with pytest.raises(MetaMorphB200Error, match="ldw%16"):
            call(name, *gemm_args(256, 264, 2, a))
        with pytest.raises(MetaMorphB200Error, match="scales missing"):
            call(name, *gemm_args(256, 256, 2, n))
        with pytest.raises(MetaMorphB200Error, match="scales missing"):
            call(name, *gemm_args(256, 256, 1, a))
        with pytest.raises(MetaMorphB200Error, match="4-byte aligned"):
            call(name, *gemm_args(256, 256, 2, c_void_p(258)))
    for name in ("mm_weight_quant_fp8", "mm_weight_dequant_fp8"):
        with pytest.raises(MetaMorphB200Error, match="multiple of 128"):
            call(name, a, ll(200), a, ll(200), a, ll(2), c_int(4), c_int(200), n)
        with pytest.raises(MetaMorphB200Error, match="null pointer"):
            call(name, a, ll(256), a, ll(256), n, ll(2), c_int(4), c_int(256), n)
        with pytest.raises(MetaMorphB200Error, match="row strides"):
            call(name, a, ll(256), a, ll(256), a, ll(1), c_int(4), c_int(256), n)
