"""CPU-only: the dG preparation entry (b200asr_f16x3_split_dg) rejects invalid arguments before any CUDA call."""
from ctypes import c_void_p


def test_split_dg_error_convention_without_gpu(pkg):
    lib = pkg.load_library()
    p = c_void_p(256)                     # never dereferenced: every call below fails its argument checks
    rc = lib.b200asr_f16x3_split_dg(None, 2, 128, 2048, p, p, p, p, p, p, p, None)
    assert rc == -1 and "null pointer" in pkg.lib.last_error()
    rc = lib.b200asr_f16x3_split_dg(p, 2, 128, 2048, p, p, p, p, None, p, p, None)
    assert rc == -1 and "all of hi, lo and sinv" in pkg.lib.last_error()
    for ndir, rows, cols in [(3, 128, 2048), (0, 128, 2048), (2, 0, 2048), (2, 128, 0), (2, 128, 2046)]:
        rc = lib.b200asr_f16x3_split_dg(p, ndir, rows, cols, p, p, p, None, None, None, p, None)
        assert rc == -1 and "f16x3_split_dg" in pkg.lib.last_error(), (ndir, rows, cols)
