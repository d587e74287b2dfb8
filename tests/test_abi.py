"""CPU tests: the C-ABI library builds for sm_90a (H100), loads, and exports every symbol that
include/pic_b200.h declares (no compute calls without a GPU)."""
import ctypes as C
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    src = open(os.path.join(ROOT, "include", "pic_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(pic_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_are_exported():
    from warpx_b200 import build
    path = build.build()          # nvcc cross-compiles sm_90a without a GPU
    L = C.CDLL(path)
    names = declared_functions()
    assert len(names) >= 18
    for n in names:
        assert hasattr(L, n), n
    L.pic_version.restype = C.c_char_p
    assert b"sm_90a" in L.pic_version()
    # every device image in the library is sm_90a code (an image for another architecture does not load on an H100)
    import subprocess
    cuobjdump = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    elves = subprocess.run([cuobjdump, "--list-elf", path], capture_output=True, text=True, check=True).stdout.split()
    cubins = [e for e in elves if e.endswith(".cubin")]
    assert cubins and all(e.endswith(".sm_90a.cubin") for e in cubins), cubins


def test_ctypes_mirror_matches_header_layout():
    """abi.py struct sizes == what the C compiler lays out for include/pic_b200.h."""
    import subprocess
    import tempfile
    from warpx_b200 import abi
    code = '#include <stdio.h>\n#include "pic_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(pic_fab), sizeof(pic_soa), sizeof(pic_stencil), sizeof(pic_bins), sizeof(pic_geom), sizeof(pic_escape_list), sizeof(pic_boundaries), sizeof(pic_laser_antenna), sizeof(pic_plasma_injector));return 0;}\n'
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "s.c")
        open(src, "w").write(code)
        exe = os.path.join(d, "s")
        subprocess.run(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe], check=True)
        sizes = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert sizes == [C.sizeof(abi.pic_fab), C.sizeof(abi.pic_soa), C.sizeof(abi.pic_stencil),
                     C.sizeof(abi.pic_bins), C.sizeof(abi.pic_geom), C.sizeof(abi.pic_escape_list),
                     C.sizeof(abi.pic_boundaries), C.sizeof(abi.pic_laser_antenna), C.sizeof(abi.pic_plasma_injector)]


def test_no_cpu_fallback():
    """The product refuses to run without a CUDA device instead of silently using the oracle."""
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from warpx_b200 import engine
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        engine.Simulation((8, 8, 8), (0, 0, 0), (1, 1, 1), nox=1)


def test_product_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "warpx_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"import\s+oracle|from\s+oracle|oracle/|oracle\.|libpic_oracle|orc_[a-z]", txt), \
                    os.path.join(dirpath, f)


def test_library_is_current_by_content_not_by_time(monkeypatch):
    """A copied or re-checked-out tree (new modification times) keeps using the library build() made; other sources
    or flags make it stale."""
    from warpx_b200 import build
    build.build()
    assert not build.stale()
    later = os.path.getmtime(build.LIB) + 100
    for f in build.sources():
        os.utime(f, (later, later))
    assert not build.stale()
    monkeypatch.setattr(build, "digest", lambda: "0" * 64)
    assert build.stale()
