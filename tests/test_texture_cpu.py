"""CPU suite: the texture checks of tests/test_texture_gpu.py on the host build of the device headers (tools/cpu_emu).

The emulator answers rb_texture_test with the same tex_eval / tex_eval_channels / d_tex_eval, compiled by g++ (no FMA contraction,
IEEE division and square root) and with a single-lane scatter of plain adds.  Every family, lane pattern and exact-sum case of the GPU
module runs here, the largest batches cut to 2^16 lookups.

Run as a script (`python tests/test_texture_cpu.py <emulator.so> <group>`) this file is also the subprocess that binds the emulator in
place of the library."""
import ctypes
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GROUPS = ["lookup_scale0", "lookup_scale1", "lookup_scale2", "lanes", "exact", "arguments"]


@pytest.fixture(scope="module")
def emulator():
    from test_device_code_cpu import _build
    return _build()


@pytest.mark.parametrize("group", GROUPS)
def test_emulator_texture_lookups_against_float64(emulator, group):
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
    import test_texture_gpu as t
    dev = torch.device("cpu")
    cap = 1 << 16
    if group.startswith("lookup_scale"):
        for tex in t.TEXTURES + [(0, 0, c) for c in t.CONSTANTS]:
            t.check_texture(rb, dev, tex, int(group[-1]), n=256)
    elif group == "lanes":
        for tex, pattern, n in t.LANE_CASES:
            t.check_lanes(rb, dev, tex, pattern, min(n, cap))
    elif group == "exact":
        for tex, n in t.EXACT_CASES:
            t.check_exact(rb, dev, tex, min(n, cap))
    else:
        t.check_arguments(rb, dev, _lib._lib, _lib.last_error, device_checks=False)
    print("ok", group, flush=True)


if __name__ == "__main__":
    main()
