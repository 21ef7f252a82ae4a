"""CPU suite: the ray-query checks of tests/test_bvh_gpu.py on the host build of the device headers (tools/cpu_emu).

The emulator builds a median-split tree in the library's node format and answers rb_scene_trace_rays with the same traversal and the same
brute force (rb_bvh.cuh).  On a few small scenes of the GPU module, the traversal must equal brute force and the float64 closest hit, as
there.  The structure checks are specific to the GPU's LBVH builder and stay in the GPU module.

Run as a script (`python tests/test_bvh_cpu.py <emulator.so> <scene>...`) this file is also the subprocess that binds the emulator in
place of the library."""
import ctypes
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

CPU_SCENES = ["soup_2000", "morton_ties", "soup_far", "soup_small", "soup_negative", "slivers", "one_triangle", "two_triangles", "three_triangles",
              "multi_shape", "depth_63"]


@pytest.fixture(scope="module")
def emulator():
    from test_device_code_cpu import _build
    return _build()


@pytest.mark.parametrize("name", CPU_SCENES)
def test_emulator_traversal_equals_brute_force_and_float64(emulator, name):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), emulator, name], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "ok " + name in r.stdout.splitlines(), r.stdout


def test_trace_rays_rejects_bad_arguments(emulator):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), emulator, "--arguments"], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "ok arguments" in r.stdout.splitlines(), r.stdout


def main():
    so, names = sys.argv[1], sys.argv[2:]
    sys.path.insert(0, HERE)
    sys.path.insert(0, ROOT)
    import torch
    from redner_b200 import _lib
    _lib._lib = _lib._bind(ctypes.CDLL(so))  # this process only: the emulator exports the same C ABI with host pointers
    from redner_b200 import redner as rb
    import test_bvh_gpu as t
    dev = torch.device("cpu")
    for name in names:
        if name == "--arguments":
            scene, _ = t.make_scene(t.SCENES["two_triangles"](), dev, rb)
            with pytest.raises(ValueError):
                scene.trace_rays(torch.zeros(4, 7))
            lib = _lib._lib
            assert lib.rb_scene_trace_rays(scene._handle, None, -1, 0, None, None) == 1
            assert "negative number of rays" in _lib.last_error(lib)
            assert lib.rb_scene_trace_rays(None, None, 0, 0, None, None) == 1
            assert "null scene" in _lib.last_error(lib)
            ids, tt = scene.trace_rays(torch.zeros(0, 8))
            assert ids.shape == (0, 2) and tt.shape == (0,)
            print("ok arguments", flush=True)
            continue
        scene, shapes = t.make_scene(t.SCENES[name](), dev, rb)
        t.check_queries(name, scene, shapes, dev, n=200, n_aim=1400, n_f64=400)
        print("ok", name, flush=True)


if __name__ == "__main__":
    main()
