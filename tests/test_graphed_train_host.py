"""CPU-only checks of the capture-safe overflow entry point (no device call is made)."""
import os


def test_overflow_accumulate_validates_its_pointers():
    from graph_pde_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    L = _lib.lib()
    assert L.nnconv_overflow_accumulate(None, None, None) != _lib.OK
    assert b'null pointer' in L.nnconv_last_error()
