"""CPU: the C-ABI library loads and exports every symbol declared in include/muon_b200.h."""
import os
import re

from conftest import ROOT


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "muon_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mub_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported_and_bound():
    from muon_b200 import _lib
    lib = _lib.load()
    syms = declared_symbols()
    assert len(syms) >= 16
    bound = set(_lib.SIGNATURES) | set(_lib.SPECIAL_RESTYPE)
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in the header but not exported by the .so"
        assert s in bound, f"{s} declared in the header but has no ctypes signature"
    assert bound <= set(syms), f"bound but undeclared: {bound - set(syms)}"


def test_version_and_error_string():
    from muon_b200 import _lib
    lib = _lib.load()
    assert lib.mub_version() >= 100
    assert isinstance(lib.mub_last_error(), (bytes, type(None)))
    assert lib.mub_gram_workspace_bytes(0, 64) == 0


def test_built_for_sm90a():
    import shutil
    import subprocess
    from muon_b200._lib import LIB_PATH
    tool = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    if not os.path.isfile(tool):
        return
    out = subprocess.run([tool, "--list-elf", LIB_PATH], capture_output=True, text=True)
    if out.returncode == 0:
        assert "sm_90a" in out.stdout
