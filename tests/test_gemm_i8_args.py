"""CPU: the B2L_F_GEMM_I8 weight source of the prefill GEMM (b2l_q4_gemm, b2l_w8_gemm and their _nll forms): the flag
values agree between include/b2l.h and _lib.py, and every combination the kernel cannot run is rejected with a message
naming the entry point and the flag before anything touches the device."""
import ctypes as C
import os
import re

import pytest

import __graft_entry__ as entry

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FNS = ["b2l_q4_gemm", "b2l_w8_gemm", "b2l_q4_gemm_nll", "b2l_w8_gemm_nll"]


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


P = 1 << 20   # 16-byte aligned, never dereferenced: every call below fails its argument checks first


def _call(L, fn, **kw):
    a = dict(x=P, ldx=1024, qw_tiled=P, scales=P, zeros=P, sz_dtype=L.B2L_BF16, y=P, ldy=256, M=64, N=256, K=1024,
             prologue=L.PRO_NONE, norm_scale=None, eps=1e-5, epilogue=L.EPI_STORE, res=None, ldres=0, split_k=0, flags=0)
    a.update(kw)
    args = L.Q4LinearArgs(**a)
    lib = L.lib()
    if fn.endswith("_nll"):
        # nll args that fail their own checks: a call that passes the flag checks stops there, still before any launch
        nl = L.NLLArgs(targets=None, targets_i64=0, nll=None, nll_sum=None, workspace=None)
        rc = getattr(lib, fn)(C.byref(args), C.byref(nl), None)
    else:
        rc = getattr(lib, fn)(C.byref(args), None)
    return rc, lib.b2l_last_error().decode()


def test_flag_values_match_the_header(L):
    h = open(os.path.join(ROOT, "include", "b2l.h")).read()
    for name, want in (("GEMM_I8", 4096), ("GEMM_I8_LO", 8192), ("GEMM_I8_HI", 16384)):
        assert re.search(rf"B2L_F_{name} = {want}\b", h), name
        assert getattr(L, "F_" + name) == want
    # the next free bits after B2L_F_STEPWISE, distinct from every other flag
    others = [int(v) for n, v in re.findall(r"B2L_F_(\w+) = (\d+)", h) if not n.startswith("GEMM_I8")]
    assert max(others) == L.F_STEPWISE == 2048 and L.F_GEMM_I8 == 2 * L.F_STEPWISE


@pytest.mark.parametrize("fn", FNS)
def test_bad_flag_combinations_are_rejected(L, fn):
    I8, LO, HI = L.F_GEMM_I8, L.F_GEMM_I8_LO, L.F_GEMM_I8_HI
    rc, msg = _call(L, fn, flags=I8 | LO | HI)
    assert rc == -1 and fn in msg and "B2L_F_GEMM_I8_LO and B2L_F_GEMM_I8_HI" in msg, msg
    for half in (LO, HI):
        rc, msg = _call(L, fn, flags=half)
        assert rc == -1 and fn in msg and "need B2L_F_GEMM_I8" in msg, msg
    for flags in (L.F_PDL, 2, 4, 64, L.F_STEPWISE, 1 << 15, 1 << 20, I8 | L.F_PDL, I8 | LO | (1 << 15)):
        rc, msg = _call(L, fn, flags=flags)
        assert rc == -2 and fn in msg and "unknown flags" in msg, (flags, msg)
    # a half of an interleaved tiling is whole 8-row groups
    for N in (200 + 4, 8 * 16 + 1):
        for half in (LO, HI):
            rc, msg = _call(L, fn, flags=I8 | half, N=N, ldy=N)
            assert rc == -2 and fn in msg and "B2L_F_GEMM_I8_LO / _HI" in msg and "multiple of 8" in msg, (N, msg)


@pytest.mark.parametrize("fn", FNS)
def test_good_flags_pass_the_flag_checks(L, fn):
    """Every accepted source reaches the checks after the flags: here the null nll arguments (the _nll forms) or, for
    the plain forms, a prologue the GEMM does not have."""
    for flags in (0, L.F_GEMM_I8, L.F_GEMM_I8 | L.F_GEMM_I8_LO, L.F_GEMM_I8 | L.F_GEMM_I8_HI):
        if fn.endswith("_nll"):
            rc, msg = _call(L, fn, flags=flags, N=200, ldy=200)
            assert rc == -1 and fn in msg and "flags" not in msg and "B2L_F_" not in msg, (flags, msg)
        else:
            rc, msg = _call(L, fn, flags=flags, N=200, ldy=200, prologue=L.PRO_RMSNORM, norm_scale=P)
            assert rc == -2 and "plain linear only" in msg, (flags, msg)
