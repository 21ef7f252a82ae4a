"""CPU suite: the environment-map checks of tests/test_envmap_gpu.py on the host build of the device headers (tools/cpu_emu).

The emulator answers rb_envmap_test with the same envmap_eval / d_envmap_eval / envmap_sample / envmap_pdf, compiled by g++ (no FMA
contraction, IEEE division and square root) and with a single-lane scatter of plain adds.  Every map, transform, family and lane
pattern of the GPU module runs here, with fewer queries per family and the largest exact batch cut to 2^16.

Run as a script (`python tests/test_envmap_cpu.py <emulator.so> <group>`) this file is also the subprocess that binds the emulator in
place of the library."""
import ctypes
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MAPS = ["1x1", "1x2", "2x1", "5x13", "16x32", "zero_rows_cols", "hot_texel", "last_row", "1024x2048"]
GROUPS = ["lookup_" + m for m in MAPS] + ["samples", "exact", "arguments"]


@pytest.fixture(scope="module")
def emulator():
    from test_device_code_cpu import _build
    return _build()


@pytest.mark.parametrize("group", GROUPS)
def test_emulator_envmap_against_float64(emulator, group):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), emulator, group], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-4000:]
    assert "ok " + group in r.stdout.splitlines(), r.stdout[-3000:]


def main():
    so, group = sys.argv[1], sys.argv[2]
    sys.path.insert(0, HERE)
    sys.path.insert(0, ROOT)
    import torch
    from redner_b200 import _lib
    _lib._lib = _lib._bind(ctypes.CDLL(so))  # this process only: the emulator exports the same C ABI with host pointers
    from redner_b200 import redner as rb
    import test_envmap_gpu as t
    dev = torch.device("cpu")
    if group.startswith("lookup_"):
        for xform in t.XFORMS:
            t.check_lookups(rb, dev, group[len("lookup_"):], xform, n=64)
    elif group == "samples":
        for m in t.MAPS:
            for xform in t.XFORMS:
                t.check_samples(rb, dev, m, xform)
    elif group == "exact":
        for n in t.EXACT_CASES:
            t.check_exact(rb, dev, min(n, 1 << 16))
    else:
        t.check_arguments(rb, dev, _lib._lib, _lib.last_error, device_checks=False)
    print("ok", group, flush=True)


if __name__ == "__main__":
    main()
