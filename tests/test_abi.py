"""CPU-side checks of the boundary: the shared library loads, exports every symbol the header declares, and the
pure host helpers (grids, base-case size) agree with the oracle restatement.  No compute calls (no GPU here)."""
import os, re
import pytest
import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "capital_b200.h")).read()
    declared = set(re.findall(r"\b(capital_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(_lib.EXPORTS)
    L = _lib.lib()
    for name in declared:
        assert hasattr(L, name), name


@pytest.mark.parametrize("size,c", [(1, 1), (8, 2), (27, 3), (64, 4)])
def test_square_grid_matches_reference_mapping(size, c):
    for rank in range(size):
        t = cb.topo.square(size, rank, c)
        o = co.topo_square(size, rank, c)
        assert (t.d, t.x, t.y, t.z) == (o["d"], o["x"], o["y"], o["z"])


@pytest.mark.parametrize("size,c", [(1, 1), (8, 1), (8, 2), (16, 2), (4, 1)])
def test_rect_grid_matches_reference_mapping(size, c):
    for rank in range(size):
        t = cb.topo.rect(size, rank, c)
        o = co.topo_rect(size, rank, c)
        assert (t.d, t.x, t.y, t.z) == (o["d"], o["x"], o["y"], o["z"])


def test_invalid_grids_are_rejected():
    with pytest.raises(_lib.CapitalError):
        cb.topo.square(4, 0, 1, layout=1)
    with pytest.raises(_lib.CapitalError):
        cb.topo.square(6, 0, 2)  # 6 != c d d
    with pytest.raises(_lib.CapitalError):
        cb.topo.rect(6, 0, 2)


@pytest.mark.parametrize("L,c,d,bcm", [(16384, 1, 1, -5), (32768, 2, 2, -4), (64, 2, 2, -1), (96, 1, 1, -2), (100, 1, 1, 3), (7, 1, 1, -9)])
def test_bc_dimension(L, c, d, bcm):
    assert _lib.lib().capital_cholinv_bc_dimension(L, c, d, bcm) == co.bc_dimension(L, c, d, bcm)


def test_cholinv_info_validates_like_the_reference_asserts():
    with pytest.raises(ValueError):
        cb.cholinv.info(1, 0, 0, "U")
    with pytest.raises(ValueError):
        cb.cholinv.info(1, 1, 0, "L")


def test_peer_wait_mode_without_a_clique():
    # -1 = "this context has not joined a clique" (also for NULL): no compute, no GPU needed
    assert _lib.lib().capital_peer_wait_mode(None) == -1


def test_experimental_tf32_entry_points_reject_a_null_context():
    import ctypes as C
    L = _lib.lib()
    n, f = C.c_int64(), C.c_double()
    assert L.capital_set_trailing_precision(None, 1) == _lib.ERR_INVALID
    assert L.capital_tf32_stats(None, C.byref(n), C.byref(f)) == _lib.ERR_INVALID
    assert L.capital_blas_gemm_tn_tf32(None, 1, 1, 1, 1.0, None, 1, None, 1, 0.0, None, 1, 0, 1) == _lib.ERR_INVALID


def test_create_fails_loudly_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    g = cb.topo.square(1, 0, 1).grid
    with pytest.raises(_lib.CapitalError):
        _lib.Context(g, 0)


def test_plain_c_caller_compiles_and_links():
    """examples/cholinv_driver.c is the reference's bench main re-written against the C ABI in plain C: it must compile with gcc
    (no CUDA headers) and link against the shared library; without a GPU it must fail loudly, not fall back."""
    import subprocess, tempfile
    exe = os.path.join(tempfile.mkdtemp(), "cholinv_driver")
    libdir = os.path.join(ROOT, "capital_b200")
    r = subprocess.run(["gcc", "-O2", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "cholinv_driver.c"),
                        "-L" + libdir, "-lcapital_b200", "-Wl,-rpath," + libdir, "-lm", "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    import torch
    if not torch.cuda.is_available():
        run = subprocess.run([exe, "128", "1", "1", "1", "-1", "0", "0", "1"], capture_output=True, text=True)
        assert run.returncode == 1 and "no sm_90 device" in run.stderr


def test_product_path_never_touches_the_oracle():
    """oracle/ is test infrastructure: the package (product path) must not import, link or execute anything under it, and the
    library must not silently fall back to a CPU path (capital_create refuses anything but an sm_90 device)."""
    import glob
    pkg = os.path.join(ROOT, "capital_b200")
    for path in glob.glob(os.path.join(pkg, "*.py")) + glob.glob(os.path.join(pkg, "csrc", "*.cu*")):
        if os.path.basename(path) == "build.py":
            continue
        src = open(path).read()
        assert "oracle" not in src.replace("the oracle", ""), path
    api = open(os.path.join(pkg, "csrc", "api.cu")).read()
    assert "prop.major != 9" in api and "no fallback" in api
