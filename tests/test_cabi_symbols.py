"""The C-ABI library loads on a machine without a GPU and exports every symbol include/nvrx_snap.h declares."""
import ctypes
import re
from pathlib import Path

from conftest import ROOT


def declared_functions():
    text = (ROOT / "include" / "nvrx_snap.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(nvrx_[a-z0-9_]+)\s*\(", text)))


def test_header_and_binding_agree():
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    assert declared_functions() == sorted(_cabi.EXPORTED_SYMBOLS)


def test_library_exports_every_symbol(built_library):
    lib = ctypes.CDLL(str(built_library))
    for name in declared_functions():
        assert hasattr(lib, name), f"{name} missing from {built_library}"


def test_library_loads_through_binding_and_reports_abi(built_library):
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    lib = _cabi.lib()
    assert lib.nvrx_abi_version() == _cabi.ABI_VERSION
    assert _cabi.strerror(0) == "ok"
    assert "invalid" in _cabi.strerror(_cabi.E_INVALID)


def test_library_is_sm90a_only(built_library):
    import shutil
    import subprocess

    if shutil.which("cuobjdump") is None:
        return
    out = subprocess.run(["cuobjdump", "-lelf", str(built_library)], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_no_oracle_in_product():
    """The product tree must not import or reference the oracle (it is test infrastructure)."""
    bad = []
    for path in (ROOT / "nvidia-resiliency-ext_b200").rglob("*"):
        if path.suffix in (".py", ".cu", ".cuh", ".h", ".cpp") and path.is_file():
            if re.search(r"\boracle\b", path.read_text(errors="ignore")):
                bad.append(str(path))
    assert not bad, bad


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    monkeypatch.setenv("NVRX_B200_LIB", str(tmp_path / "nope.so"))
    monkeypatch.setattr(_cabi, "_LIB", None)
    try:
        _cabi.lib()
    except _cabi.SnapError as e:
        assert "no CPU fallback" in str(e)
    else:
        raise AssertionError("expected SnapError")
