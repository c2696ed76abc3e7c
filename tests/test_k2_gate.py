"""The error-word gate of the k2 chain on the device (csrc/k2_history_kernel.cuh): wva_ingest_v2's analyze graph cannot
read the keys pass's error word back before the history would change, so k2_resolve_kernel and k2_slot_kernel test it
themselves.  wva_ingest_v2_create checks the registry the keys pass checks, so no cycle through the public API sets the
word; tests/device_prims/k2_gate.cu runs the product's kernels directly with the word clear and set."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gate(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("k2_gate") / "libk2gate.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "--fmad=false", "-std=c++17", "-Xcompiler",
                    "-fPIC", "-shared", "-o", so, os.path.join(ROOT, "tests", "device_prims", "k2_gate.cu"), "-lcudart"],
                   check=True)
    lib = C.CDLL(so)

    def run(err):
        cnt, vals = np.full(3, -7, np.int32), np.full(30, -7.0)
        eff, k2 = np.full(1, -7, np.int64), np.full(4, -7, np.int64)
        assert lib.k2_gate(C.c_int(err), *(x.ctypes.data_as(C.c_void_p) for x in (cnt, vals, eff, k2))) == 0
        return cnt, vals, eff, k2
    return run


def test_clear_word_runs_the_chain(gate):
    cnt, vals, eff, k2 = gate(0)
    assert cnt.tolist() == [3, 0, 0]                          # three observations of (accelerator 0, "short")
    assert vals[:3].tolist() == [500.0, 600.0, 700.0]
    assert k2.tolist() == [500, 600, 550, 700]                # the unobserved replica averages the two before it
    assert eff[0] == 700                                      # the slot's last data replica: min(k1 = 800, 700)


@pytest.mark.parametrize("err", [1, 2])
def test_set_word_leaves_history_and_slot_untouched(gate, err):
    cnt, vals, eff, k2 = gate(err)
    assert cnt.tolist() == [0, 0, 0] and not vals.any()      # the history as it was (empty)
    assert eff[0] == 0                                        # the slot kernel wrote nothing either
