"""The C-ABI library loads and exports exactly what include/dmosopt_b200.h declares (no GPU needed)."""

import ctypes
import os
import re
import shutil
import subprocess

import pytest

from conftest import ROOT

HEADER = os.path.join(ROOT, "include", "dmosopt_b200.h")


def header_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dmo_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib_path():
    from dmosopt_b200 import build

    return build.build(verbose=False)


def test_header_declares_the_documented_surface():
    syms = header_symbols()
    for s in ("dmo_create", "dmo_rank_nd", "dmo_crowding_distance", "dmo_remove_worst", "dmo_tournament", "dmo_nsga2_generate",
              "dmo_gp_create", "dmo_gp_predict", "dmo_hypervolume", "dmo_ehvi_select", "dmo_get_duplicates"):
        assert s in syms


def test_library_exports_every_header_symbol(lib_path):
    lib = ctypes.CDLL(lib_path)
    for s in header_symbols():
        assert hasattr(lib, s), f"{s} declared in the header but not exported"
    assert lib.dmo_version() >= 100


def test_python_binding_covers_every_header_symbol(lib_path):
    from dmosopt_b200 import _lib

    assert sorted(_lib._SIGNATURES) == header_symbols()
    _lib.load_library()  # declares all prototypes; raises if a symbol is missing


def test_library_is_built_for_sm_90a(lib_path):
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    out = subprocess.run([cuobjdump, "-lelf", lib_path], capture_output=True, text=True).stdout
    cubins = re.findall(r"\.(sm_\w+)\.cubin", out)
    assert cubins and set(cubins) == {"sm_90a"}, out


def test_no_gpu_means_loud_failure(lib_path):
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from dmosopt_b200 import _lib

    with pytest.raises(_lib.DmoError):
        _lib.rank_nd([[0.0, 1.0], [1.0, 0.0]])


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "dmosopt_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, flags=re.M), f


def test_plain_c_host_compiles_and_links_against_the_header(lib_path, tmp_path):
    """include/dmosopt_b200.h is valid C99 and examples/nsga2_step.c (a non-Python host of the fused generation step)
    links against the shared library with nothing but gcc; without a GPU the program stops at dmo_create."""
    import shutil
    import subprocess

    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "nsga2_step")
    libdir = os.path.dirname(lib_path)
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(root, "include"), os.path.join(root, "examples", "nsga2_step.c"),
                        "-L", libdir, "-ldmosopt_b200", f"-Wl,-rpath,{libdir}", "-lm", "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    import torch

    run = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    if torch.cuda.is_available():
        assert run.returncode == 0 and "generation 4:" in run.stdout, run.stdout + run.stderr
    else:
        assert run.returncode != 0 and "dmo_create" in run.stderr
