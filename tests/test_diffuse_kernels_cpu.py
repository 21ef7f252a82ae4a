"""CPU check of the diffuse-only instantiation of the kernels (rb_kernels_diffuse.cu, RB_DIFFUSE): the host build of the device
headers is compiled with -DRB_LEAN, as the lean kernels are, and once more with -DRB_LEAN -DRB_DIFFUSE.  Folding the material flags
of diffuse-only scenes into constants must not move a bit: on C1, C2, C2 with every vertex differentiable and the bunny box with
diffuse materials, both builds give the same image and the same gradients, bit for bit.  A material that computes specular
lighting, uses vertex colours or has a normal map must not reach the diffuse-only code: the library then runs the lean kernels,
and the diffuse-only host build refuses to render.  The GPU twin is tests/test_diffuse_kernels_gpu.py.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from test_device_code_cpu import _build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SAME = ["c1", "c2", "c2_all_vertices", "bunny_box_diffuse"]
FALLBACK = ["triangle_with_specular", "triangle_with_vertex_color", "triangle_with_normal_map"]


def _dump(so, names, tmp_path, tag):
    out = str(tmp_path / (tag + ".npz"))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "diffuse_check.py"), so, out] + names, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return dict(np.load(out))


@pytest.fixture(scope="module")
def outputs(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("diffuse")
    lean = _dump(_build("-DRB_LEAN"), SAME + FALLBACK, tmp, "lean")
    diffuse = _dump(_build("-DRB_LEAN -DRB_DIFFUSE"), SAME + FALLBACK, tmp, "diffuse")
    return lean, diffuse


@pytest.mark.parametrize("name", SAME)
def test_diffuse_build_is_bit_identical_to_the_lean_build(outputs, name):
    lean, diffuse = outputs
    keys = sorted(k for k in lean if k.startswith(name + "/"))
    assert name + "/image" in keys and any("/grad." in k for k in keys), keys
    assert keys == sorted(k for k in diffuse if k.startswith(name + "/"))
    assert float(np.abs(lean[name + "/image"]).sum()) > 0
    for k in keys:
        assert np.array_equal(lean[k], diffuse[k]), (k, float(np.abs(lean[k] - diffuse[k]).max()))


@pytest.mark.parametrize("name", FALLBACK)
def test_material_features_are_not_served_by_the_diffuse_build(outputs, name):
    lean, diffuse = outputs
    assert name + "/image" in lean and name + "/error" not in lean
    assert "serves diffuse-only materials" in str(diffuse.get(name + "/error", "")), sorted(k for k in diffuse if k.startswith(name))
