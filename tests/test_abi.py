"""The C-ABI library loads and exports every symbol include/psalm_b200.h declares (no compute)."""
import os
import re

import pytest

from conftest import ROOT


def _declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "psalm_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(psalm_[a-z0-9_]+)\s*\(", hdr)))


def test_header_declares_entry_points():
    syms = _declared_symbols()
    assert "psalm_msda_forward" in syms and "psalm_abi_version" in syms


def test_library_exports_every_declared_symbol():
    from psalm_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        from psalm_b200 import build
        build.build()
    h = _lib.lib()
    for s in _declared_symbols():
        assert hasattr(h, s), "libpsalm_b200.so does not export %s" % s
        assert s in _lib.SIGNATURES, "psalm_b200/_lib.py has no ctypes signature for %s" % s
    for s in _lib.SIGNATURES:
        assert s in _declared_symbols(), "%s bound in _lib.py but not declared in the header" % s
    assert h.psalm_abi_version() == 1
    assert h.psalm_compiled_arch() == 90


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from psalm_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.PsalmKernelError):
        _lib.lib()


def test_cpu_tensors_are_rejected():
    """No CPU fallback: the op raises like the reference's ms_deform_attn.h:43."""
    import torch
    from psalm_b200 import msda
    v = torch.zeros(1, 4, 1, 4)
    loc = torch.zeros(1, 2, 1, 1, 1, 2)
    w = torch.zeros(1, 2, 1, 1, 1)
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        msda.ms_deform_attn_forward(v, [(2, 2)], [0], loc, w, 128)
    with pytest.raises(NotImplementedError):
        msda.ms_deform_attn_backward()
