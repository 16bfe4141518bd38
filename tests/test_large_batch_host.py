"""CPU tests of the LM decode limits above 64 rows: the activation padding of the wide GEMM and the max_rows range that
acb_lm_create checks before any CUDA call (no GPU needed)."""
import ctypes as C

from audiocraft_b200 import _lib, build


def _L():
    build.build()
    return _lib.lib()


def test_rows_pad_values():
    L = _L()
    assert [L.acb_lm_rows_pad(r) for r in (1, 8, 16, 17, 32, 33, 64)] == [16, 16, 16, 32, 32, 64, 64]   # unchanged up to 64
    assert [L.acb_lm_rows_pad(r) for r in range(65, 129)] == [128] * 64
    assert [L.acb_lm_rows_pad(r) for r in range(129, 257)] == [256] * 128
    assert L.acb_lm_rows_pad(257) == -1                     # ACB_ERR_INVALID
    assert b'257' in L.acb_last_error()
    assert _lib.ACB_LM_MAX_ROWS == 256


def test_create_rejects_257_rows_without_a_gpu():
    L = _L()
    cfg = _lib.LMConfig(256, 4, 3, 1024, 4, 128, 1, 257, 64, 8, 1.0, 0)
    handle = C.c_void_p()
    rc = L.acb_lm_create(C.byref(cfg), C.byref(_lib.LMWeights()), C.byref(_lib.LMBuffers()), C.byref(handle))
    assert rc == -1 and handle.value is None              # ACB_ERR_INVALID, checked before any CUDA call
    assert 'max_rows 257 not in [1,256]' in L.acb_last_error().decode()
