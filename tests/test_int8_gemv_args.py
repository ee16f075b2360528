"""CPU: b2l_q8_gemv_cb (the batch-1 llm.int8 linear reading CB directly) rejects bad arguments with a message before it
touches the device."""
import ctypes as C

import pytest

import __graft_entry__ as entry


@pytest.fixture(scope="module")
def lib():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib.lib()


def test_bad_arguments_are_rejected_with_a_message(lib):
    p = C.c_void_p(1 << 20)   # 16-byte aligned, never dereferenced: every call below fails its argument checks first
    N, K = 256, 1024

    def call(x=p, cb=p, scb=p, mask=None, y=p, n=N, k=K, flags=0):
        return lib.b2l_q8_gemv_cb(x, cb, scb, mask, y, n, k, 6.0, flags, None)

    for kw in ("x", "cb", "scb", "y"):
        assert call(**{kw: None}) == -1 and b"null pointer" in lib.b2l_last_error(), kw
    assert call(k=1000) == -2 and b"multiple of 128" in lib.b2l_last_error()
    assert call(k=0) == -2 and b"multiple of 128" in lib.b2l_last_error()
    assert call(k=32768 + 128) == -2 and b"<= 32768" in lib.b2l_last_error()
    assert call(n=0) == -1 and b"bad shape" in lib.b2l_last_error()
    assert call(n=-16) == -1 and b"bad shape" in lib.b2l_last_error()
    assert call(x=C.c_void_p((1 << 20) + 8)) == -1 and b"16-byte aligned" in lib.b2l_last_error()
    assert call(cb=C.c_void_p((1 << 20) + 4)) == -1 and b"16-byte aligned" in lib.b2l_last_error()
    assert call(flags=2) == -2 and b"unknown flags" in lib.b2l_last_error()
    assert call(flags=1 | 4) == -2 and b"unknown flags" in lib.b2l_last_error()
