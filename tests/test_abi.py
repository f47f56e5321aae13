"""CPU: the C-ABI library loads, exports every symbol include/o2345.h declares, and the ctypes
table covers exactly that set (no compute calls: there is no GPU here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "o2345.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(o2345_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_something():
    assert len(declared_symbols()) >= 25


def test_library_exports_every_declared_symbol():
    from o2345 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared_symbols():
        assert hasattr(lib, name), f"{name} declared in include/o2345.h but not exported"
    assert lib.o2345_abi_version() == _lib.ABI_VERSION


def test_ctypes_table_matches_header():
    from o2345 import _lib
    assert sorted(_lib.EXPORTED) == declared_symbols()


def test_missing_library_fails_loudly(monkeypatch):
    from o2345 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libo2345_sm90.so")
    with pytest.raises(_lib.O2345Error):
        _lib.load()


def test_ops_refuse_cpu_tensors():
    import torch
    from o2345 import _lib, ops
    with pytest.raises(_lib.O2345Error):
        ops._p(torch.zeros(4))


def test_argument_checks_return_einval_without_touching_the_gpu():
    """Every entry point validates its arguments before any CUDA call: bad sizes / alignment / modes give O2345_EINVAL
    (-1) and a message through o2345_last_error -- checkable on a machine without a GPU."""
    import ctypes as C
    from o2345 import _lib
    lib = _lib.load()
    fake = C.c_void_p(0x1000)                                   # never dereferenced: the checks fail first
    ep = _lib.Epilogue(act=7)
    cases = [
        # TMA needs 16-byte row strides
        lambda: lib.o2345_gemm_f16(fake, fake, fake, 128, 128, 64, 60, 64, 128, 0, 0, 0, 0, 0, 0, 0, 0, None, None, 0, None),
        # null operand
        lambda: lib.o2345_gemm_f16(None, fake, fake, 128, 128, 64, 64, 64, 128, 0, 0, 0, 0, 0, 0, 0, 0, None, None, 0, None),
        # unknown activation
        lambda: lib.o2345_gemm_f16(fake, fake, fake, 128, 128, 64, 64, 64, 128, 0, 0, 0, 0, 0, 0, 0, 0, C.byref(ep), None, 0, None),
        # GEGLU needs N % 32 == 0
        lambda: lib.o2345_gemm_f16(fake, fake, fake, 128, 48, 64, 64, 64, 24, 0, 0, 0, 0, 0, 0, 0, 0,
                                   C.byref(_lib.Epilogue(act=3, alpha=1.0)), None, 0, None),
        # implicit conv: channels must be a multiple of 8, width must tile 128 pixels
        lambda: lib.o2345_conv3x3_f16(fake, 1, 8, 8, 12, fake, 16, fake, 16, None, None, 0, None),
        lambda: lib.o2345_conv3x3_f16(fake, 1, 8, 24, 16, fake, 16, fake, 16, None, None, 0, None),
        # attention head sizes
        lambda: lib.o2345_attention_f16(fake, fake, fake, 1, 16, 2, 48, 96, fake, 96, 1.0, None),
        # attention scale: the kernel's running maximum is only right for a positive, finite scale
        lambda: lib.o2345_attention_f16(fake, fake, fake, 1, 16, 2, 40, 240, fake, 80, 0.0, None),
        lambda: lib.o2345_attention_f16(fake, fake, fake, 1, 16, 2, 40, 240, fake, 80, -1.0, None),
        lambda: lib.o2345_attention_f16(fake, fake, fake, 1, 16, 2, 40, 240, fake, 80, float("nan"), None),
        lambda: lib.o2345_attention_f16(fake, fake, fake, 1, 16, 2, 40, 240, fake, 80, float("inf"), None),
        # softmax rows are at most 1024 long; timestep embeddings have an even width
        lambda: lib.o2345_softmax_rows(fake, 8, 1025, fake, None),
        lambda: lib.o2345_timestep_embedding(fake, 2, 321, fake, None),
        # group norm: channels not a multiple of the group count
        lambda: lib.o2345_groupnorm_stats(fake, 1, 16, 40, 32, 1e-5, None, None, fake, fake, fake, None),
        # blend precision
        lambda: lib.o2345_render_blend(C.byref(_lib.Points(mode=0)), 4, None, fake, fake, 8,
                                       C.byref(_lib.Views(V=4, H=8, W=8, maps=0x1000, proj=0x1000, centers=0x1000)), 0, fake, None,
                                       fake, 9, fake, None, None),
        # precision 2 (the wgmma kernel) was removed in ABI 5; _lib.load() refuses a library of another ABI version
        lambda: lib.o2345_render_blend(C.byref(_lib.Points(mode=0)), 4, None, fake, fake, 8,
                                       C.byref(_lib.Views(V=4, H=8, W=8, maps=0x1000, proj=0x1000, centers=0x1000)), 0, fake, None,
                                       fake, 2, fake, None, None),
    ]
    for i, call in enumerate(cases):
        rc = call()
        assert rc == -1, (i, rc, _lib.last_error())
        assert len(_lib.last_error()) > 0
