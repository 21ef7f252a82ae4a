"""CPU suite: the camera checks of tests/test_camera_gpu.py on the host build of the device headers (tools/cpu_emu).

The emulator answers rb_camera_test with the same camera_test_one, compiled by g++ (no FMA contraction, IEEE division and square root).
Every camera and family of the GPU module runs here, with fewer queries per family.

Run as a script (`python tests/test_camera_cpu.py <emulator.so> <check> <camera>`) this file is also the subprocess that binds the
emulator in place of the library."""
import ctypes
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CAMERAS = ["pinhole", "skewed", "c2w_far", "clip1", "ortho", "fisheye", "panorama", "panorama_clip0", "distort_persp", "distort_fish", "lens"]
CASES = [("rays", c) for c in CAMERAS] + [("project", c) for c in CAMERAS] + [("ray_adjoint", c) for c in CAMERAS] + \
        [("distort", c) for c in ("distort_persp", "distort_fish")] + [("finish", c) for c in CAMERAS]


@pytest.fixture(scope="module")
def emulator():
    from test_device_code_cpu import _build
    return _build()


@pytest.mark.parametrize("check,camera", CASES)
def test_emulator_camera_against_float64(emulator, check, camera):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), emulator, check, camera], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-4000:]
    assert "ok " + check in r.stdout.splitlines(), r.stdout[-3000:]


def main():
    so, check, camera = sys.argv[1], sys.argv[2], sys.argv[3]
    sys.path.insert(0, HERE)
    sys.path.insert(0, ROOT)
    import torch
    from redner_b200 import _lib
    _lib._lib = _lib._bind(ctypes.CDLL(so))  # this process only: the emulator exports the same C ABI with host pointers
    from redner_b200 import redner as rb
    import test_camera_gpu as t
    dev = torch.device("cpu")
    {"rays": t.check_rays, "project": t.check_project, "ray_adjoint": t.check_ray_adjoint, "distort": t.check_distort, "finish": t.check_finish}[check](rb, dev, camera, n=24)
    print("ok", check, flush=True)


if __name__ == "__main__":
    main()
