"""The C-ABI boundary: header, binding table and shared library must agree (no GPU needed)."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "nerfacc_b200.h")


def _declared():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(nfa_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from nerfacc_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "build with `make -C nerfacc_b200/csrc`"
    lib = C.CDLL(_lib.LIB_PATH)
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/nerfacc_b200.h but not exported"
    assert sorted(_lib.SIGNATURES) == names, "nerfacc_b200/_lib.py binding table out of sync with the header"
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    exported = sorted(l.split()[-1] for l in out.splitlines() if " T nfa_" in l)
    assert exported == names, "library exports symbols the header does not declare (or vice versa)"


def test_version_and_error_strings_without_gpu():
    from nerfacc_b200 import _lib
    lib = _lib.load()
    assert lib.nfa_version() == _lib.ABI_VERSION
    assert lib.nfa_error_string(0) == b"ok"
    assert b"argument" in lib.nfa_error_string(-1)
    # pure host helpers
    assert lib.nfa_occ_words(1, 128, 128, 128) == 32 ** 3
    assert lib.nfa_occ_coarse_words(1, 128, 128, 128) == 2048
    assert lib.nfa_occ_words(2, 30, 17, 5) == 2 * 8 * 5 * 2
    assert lib.nfa_march_workspace_bytes(65536, 1000) > 65536 * 8 + 1000 * 32
    assert lib.nfa_pack_info_workspace_bytes(10) >= 80
    assert lib.nfa_scan_by_key_workspace_bytes(1 << 20) > 0


def test_march_workspace_size_covers_its_parts():
    """nfa_march_workspace_bytes: header + tile sums and bases + three per-ray u32 arrays (sample / run counts,
    sample offset inside the tile) + the run pool of 32-byte records; grows with both arguments (pure host code)."""
    from nerfacc_b200 import _lib
    lib = _lib.load()
    for n_rays in (1, 31, 448, 65536, 1 << 20):
        for runs in (0, 1000, 3 * n_rays + 1024):
            b = lib.nfa_march_workspace_bytes(n_rays, runs)
            assert b >= 64 + 3 * 4 * n_rays + 32 * runs
            assert lib.nfa_march_workspace_bytes(n_rays, runs + 1) >= b + 32
            assert lib.nfa_march_workspace_bytes(n_rays + 512, runs) > b
    assert lib.nfa_march_workspace_bytes(-1, 0) == 0 and lib.nfa_march_workspace_bytes(4, -1) == 0


def test_argument_errors_do_not_need_a_gpu():
    from nerfacc_b200 import _lib
    lib = _lib.load()
    assert lib.nfa_scan_packed(-1, None, None, None, 0, 0, 0, 0, None) == -1
    assert lib.nfa_scan_packed(4, None, None, None, 0, 0, 0, 0, None) == -1
    assert lib.nfa_composite_fwd(3, 10, None, None, None, None, 0, None, None, None, 1, *([None] * 8)) == -1
    assert lib.nfa_intersect_sorted(1, None, None, 64, None, None, None, None, None) == -2  # > 32 boxes: unsupported
    assert lib.nfa_march_workspace_bytes(-5, 10) == 0

    # cone_angle rules of nfa_march / nfa_expand_samples: rejected before any pointer is read, so every other
    # pointer may be a dummy (non-null, 16-byte aligned) address
    P = 1 << 20

    def march(cone_angle, coarse=P, terminate_planes=None):
        return lib.nfa_march(64, P, P, None, None, 0.0, 1e10, 1, 32, 32, 32, P, coarse, P, P, None, None, None, 1e-3,
                             cone_angle, 1024, P, P, None, terminate_planes, None)

    def expand(cone_angle):
        return lib.nfa_expand_samples(64, 1024, P, P, 1e-3, cone_angle, 4096, P, P, P, P, None)

    for bad in (-0.004, float("nan")):
        assert march(bad) == -1 and expand(bad) == -1
    assert march(0.004, coarse=None) == -1
    assert march(0.004, terminate_planes=P) == -2  # the growing-step walk writes no terminate planes


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from nerfacc_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(ImportError, match="no CPU or PyTorch fallback"):
        _lib.load()


def test_product_never_touches_the_oracle():
    pkg = os.path.join(ROOT, "nerfacc_b200")
    for d, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(d, f)).read()
                assert "import oracle" not in text and "from oracle" not in text and "liboracle" not in text, f
                assert "host_sim" not in text or f.endswith((".cuh", ".cu")), f  # headers may mention the harness in comments
