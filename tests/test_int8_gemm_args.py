"""CPU: b2l_q8_gemm rejects bad arguments with a message before it touches the device, and
b2l_q8_gemm_workspace_bytes states the layout it needs."""
import ctypes as C

import pytest

import __graft_entry__ as entry


@pytest.fixture(scope="module")
def lib():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib.lib()


def test_workspace_bytes(lib):
    # CA int8 [M rounded up to the token tile, 16 or 128][K] | SCA fp32 [M] padded to 16 bytes | one mask bit per column
    assert lib.b2l_q8_gemm_workspace_bytes(2, 4096) == 16 * 4096 + 16 + 4096 // 8
    assert lib.b2l_q8_gemm_workspace_bytes(5, 32768) == 16 * 32768 + 32 + 32768 // 8
    assert lib.b2l_q8_gemm_workspace_bytes(17, 1024) == 128 * 1024 + 80 + 1024 // 8
    assert lib.b2l_q8_gemm_workspace_bytes(2, 4000) == 0      # K not a multiple of 128
    assert lib.b2l_q8_gemm_workspace_bytes(2, 32896) == 0     # K above 32768
    assert lib.b2l_q8_gemm_workspace_bytes(0, 4096) == 0


def test_bad_arguments_are_rejected_with_a_message(lib):
    p = C.c_void_p(1 << 20)   # 16-byte aligned, never dereferenced: every call below fails its argument checks first
    M, N, K = 4, 256, 1024
    ws = lib.b2l_q8_gemm_workspace_bytes(M, K)

    def call(x=p, ldx=K, cb=p, scb=p, work=p, work_bytes=ws, y=p, ldy=N, m=M, n=N, k=K, flags=0):
        return lib.b2l_q8_gemm(x, ldx, cb, scb, work, work_bytes, y, ldy, m, n, k, 6.0, flags, None)

    assert call(x=None) == -1 and b"null pointer" in lib.b2l_last_error()
    assert call(work=None) == -1 and b"null pointer" in lib.b2l_last_error()
    assert call(k=1000, ldx=1000) == -2 and b"multiple of 128" in lib.b2l_last_error()
    assert call(k=32768 + 128, ldx=32768 + 128) == -2 and b"<= 32768" in lib.b2l_last_error()
    assert call(m=0) == -1 and b"bad shape" in lib.b2l_last_error()
    assert call(ldx=K + 4) == -1 and b"leading dimension" in lib.b2l_last_error()
    assert call(ldy=N - 1) == -1 and b"leading dimension" in lib.b2l_last_error()
    assert call(cb=C.c_void_p((1 << 20) + 8)) == -1 and b"16-byte aligned" in lib.b2l_last_error()
    assert call(work_bytes=ws - 1) == -1 and b"too small" in lib.b2l_last_error()
    assert call(flags=1) == -2 and b"flags" in lib.b2l_last_error()
