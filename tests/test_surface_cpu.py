"""CPU suite: the geometry checks of tests/test_surface_gpu.py on the host build of the device headers (tools/cpu_emu).

The emulator answers rb_surface_test with the same surface_test_one, compiled by g++ (no FMA contraction, IEEE division and square root).
Every mesh and family of the GPU module runs here, with fewer queries per family.

Run as a script (`python tests/test_surface_cpu.py <emulator.so> <check> <mesh>`) this file is also the subprocess that binds the
emulator in place of the library."""
import ctypes
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MESHES = ["bare", "attrs", "seamed", "uvdeg", "uvdeg_flip", "normals", "near_minus_z", "scale"]
CASES = [(c, m) for c in ("point", "adjoint", "light") for m in MESHES] + [("scatter", "all"), ("errors", "all"), ("slips", "all")]


@pytest.fixture(scope="module")
def emulator():
    from test_device_code_cpu import _build
    return _build()


@pytest.mark.parametrize("check,mesh", CASES)
def test_emulator_surface_against_float64(emulator, check, mesh):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), emulator, check, mesh], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-4000:]
    assert "ok " + check in r.stdout.splitlines(), r.stdout[-3000:]


def main():
    so, check, mesh = sys.argv[1], sys.argv[2], sys.argv[3]
    sys.path.insert(0, HERE)
    sys.path.insert(0, ROOT)
    import torch
    from redner_b200 import _lib
    _lib._lib = _lib._bind(ctypes.CDLL(so))  # this process only: the emulator exports the same C ABI with host pointers
    from redner_b200 import redner as rb
    import surface_ref
    import test_surface_gpu as t
    dev = torch.device("cpu")
    if check == "point":
        t.check_point(rb, dev, mesh, n=16)
    elif check == "adjoint":
        t.check_adjoint(rb, dev, mesh, n=8)
    elif check == "light":
        t.check_light(rb, dev, mesh, n=16)
    elif check == "scatter":
        t.check_scatter(rb, dev)
    elif check == "errors":
        t.check_errors(rb, dev)
    elif check == "slips":
        terms = {}
        for m in MESHES:
            t.check_adjoint(rb, dev, m, n=4, slip_terms=terms)
        assert all(terms.get(sl, 0) > 0 for sl in surface_ref.SLIPS), terms
    print("ok", check, flush=True)


if __name__ == "__main__":
    main()
