"""The C-ABI library loads, exports every symbol include/cuba_b200.h declares, and refuses to compute
without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT


def _declared_functions():
    text = open(os.path.join(ROOT, "include", "cuba_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(cuba_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol(pkg):
    lib = ctypes.CDLL(pkg.library_path())
    names = _declared_functions()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), "libcuba_b200.so lacks %s" % n
    # the binding's list is the same set
    assert sorted(pkg.binding.exported_symbols()) == names


def test_cpp_api_symbols_present(pkg):
    import subprocess
    out = subprocess.run(["nm", "-D", "--defined-only", "-C", pkg.library_path()], capture_output=True, text=True).stdout
    assert "cuba::CudaBundleAdjustment::create()" in out
    assert "cuba::CudaBundleAdjustment::~CudaBundleAdjustment()" in out


def test_only_sm90a_code_is_embedded(pkg):
    import subprocess
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-lelf", pkg.library_path()], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_no_cpu_fallback(pkg):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(pkg.CubaError, match="no CPU fallback"):
        pkg.Engine()


KERNEL_OPTIONS = {0: "pcg_variant", 2: "jh_variant", 3: "schur_variant"}   # cuba_config.reserved[slot] <- Engine keyword


@pytest.mark.parametrize("slot,value", [(0, 1), (2, 5), (2, 6), (3, 1), (3, 2), (3, 4), (0, -1), (0, 9), (2, 10), (3, 6)])
def test_create_rejects_options_that_name_no_kernel(pkg, slot, value):
    """the values of retired kernels (k_pcg, J+H generations 2 and 3, k_schur, the tile-local Schur pair, k_schur4) and values
    out of range fail with CUBA_ERR_INVALID and a message naming the slot and the value -- before any device is touched, so the
    same on a machine without a GPU"""
    with pytest.raises(pkg.CubaError, match=r"^cuba error -1: .*reserved\[%d\] = %d " % (slot, value)):
        pkg.Engine(**{KERNEL_OPTIONS[slot]: value})


def test_create_accepts_every_option_that_names_a_kernel(pkg):
    """every value that names a kernel passes the check; without a GPU creation then fails with the no-device error"""
    for slot, values in ((0, (0, 2, 3, 4, 5, 6, 7, 8)), (2, (0, 1, 2, 3, 4, 7, 8, 9)), (3, (0, 3, 5))):
        for v in values:
            try:
                pkg.Engine(**{KERNEL_OPTIONS[slot]: v}).close()
            except pkg.CubaError as e:
                assert str(e).startswith("cuba error -2: no CUDA device"), (slot, v, str(e))


def test_product_does_not_touch_the_oracle():
    """the product package and its native sources never import / link anything under oracle/"""
    pdir = os.path.join(ROOT, "cuda-bundle-adjustment_b200")
    for dirpath, _, files in os.walk(pdir):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert "ba_oracle" not in text and "libcuba_ref" not in text, f
                assert not re.search(r"^\s*(import|from)\s+oracle", text, flags=re.M), f
