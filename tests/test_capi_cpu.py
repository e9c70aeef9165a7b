"""CPU: the C-ABI library builds, loads, and exports every symbol include/g2pc.h declares (no compute calls)."""
import ctypes
import os
import re

import pytest

from util import ROOT


def _declared_functions():
    text = open(os.path.join(ROOT, "include", "g2pc.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(g2pc_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol(lib):
    from g2pc import capi
    names = _declared_functions()
    assert "g2pc_sample_count" in names and "g2pc_sample_emit" in names
    raw = ctypes.CDLL(capi.LIB_PATH)
    for name in names:
        assert hasattr(raw, name), f"{name} declared in include/g2pc.h but not exported by libg2pc.so"
    assert sorted(capi.SIGNATURES.keys()) == names, "g2pc/capi.py bindings out of sync with include/g2pc.h"
    assert lib.g2pc_version() >= 100
    assert lib.g2pc_last_error() is not None


def test_struct_layouts_match_header():
    """g2pc_tile_t / g2pc_unit_t are 4 x int32 (the planner uploads (T,4) int32 arrays)."""
    text = open(os.path.join(ROOT, "include", "g2pc.h")).read()
    for struct in ("g2pc_tile_t", "g2pc_unit_t"):
        body = re.search(r"typedef struct \{([^}]*)\} " + struct, text).group(1)
        assert len(re.findall(r"int32_t\s+\w+;", body)) == 4


def test_missing_library_fails_loudly(tmp_path):
    from g2pc import capi
    with pytest.raises(capi.G2pcError):
        capi.load(str(tmp_path / "nope.so"))


def test_sass_is_sm90a(lib):
    """The shipped library carries sm_90a code (no PTX-JIT fallback to another arch)."""
    import shutil
    import subprocess
    from g2pc import capi
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    out = subprocess.run(["cuobjdump", "-lelf", capi.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_product_never_imports_the_oracle():
    """oracle/ is test infrastructure: nothing under 3dgs-to-pc_b200/ may import or execute it."""
    pkg = os.path.join(ROOT, "3dgs-to-pc_b200")
    offenders = []
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                text = open(os.path.join(dirpath, f), errors="replace").read()
                if re.search(r"^\s*(from|import)\s+oracle\b", text, flags=re.M) or re.search(r"import_module\(.oracle", text):
                    offenders.append(os.path.join(dirpath, f))
    assert not offenders, offenders
