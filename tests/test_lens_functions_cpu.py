"""CPU suite, function level: the thin-lens camera functions of the device headers (tests/lens_functions.cpp, compiled for the host with
Real = double) against the float64 restatement of tests/lens_ref.py and against central differences.

- concentric_disc (rb_camera.cuh) gives the known answers of Shirley-Chiu's map on a grid through its wedge boundaries, and equals the
  restatement everywhere on the grid.
- cam_sample_lens and cam_project_lens_d (near-clipped cases included) equal the restatement.
- d_cam_sample_lens and d_cam_project_lens agree with central differences w.r.t. the vertices, cam_to_world / world_to_cam, intr_inv /
  intrinsic_mat, lens_radius and focus_distance.
- The distribution invariant of primary_edge_weight (shared by the host and device builders; tests/test_lens_gpu.py shows the device
  table equals the host's): every random edge that is a silhouette from one of 10^4 lens points and whose projection from it meets the
  image has a positive weight, edges on a ray through the lens centre and edges outside the centre view but within reach of the circle
  of confusion included."""
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import lens_ref

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.isdir("/usr/local/cuda/include"):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("lens") / "lens_functions")
    cmd = ["g++", "-O2", "-std=c++17", "-w", "-DRB_REAL_DOUBLE", "-include", os.path.join(ROOT, "tools", "cpu_emu", "emu_shim.h"), "-I/usr/local/cuda/include",
           "-I" + os.path.join(ROOT, "include"), '-DRB_DATA_DIR="%s"' % os.path.join(ROOT, "redner_b200", "data"), os.path.join(HERE, "lens_functions.cpp"),
           "-o", out]
    subprocess.run(cmd, check=True, timeout=900)
    return out


def _run(exe, mode):
    r = subprocess.run([exe, mode], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    return r.stdout


def test_concentric_disc_known_answers(exe):
    rows = np.array([[float(x) for x in l.split()] for l in _run(exe, "disc").splitlines()])
    got = {(u1, u2): (x, y) for u1, u2, x, y in rows}
    h = math.sqrt(0.5)
    known = {(0.5, 0.5): (0, 0), (0.75, 0.5): (0.5, 0), (0.5, 0.75): (0, 0.5), (0.25, 0.5): (-0.5, 0), (0.5, 0.25): (0, -0.5),
             (0.75, 0.75): (0.5 * h, 0.5 * h), (0.25, 0.25): (-0.5 * h, -0.5 * h), (0.75, 0.25): (0.5 * h, -0.5 * h), (0.0, 0.5): (-1, 0),
             (0.5, 0.0): (0, -1), (0.0, 0.0): (-h, -h)}
    for u, xy in known.items():
        assert np.allclose(got[u], xy, atol=1e-15), (u, got[u], xy)
    for (u1, u2), xy in got.items():
        assert np.allclose(xy, lens_ref.concentric(u1, u2), atol=1e-15)
        assert xy[0] ** 2 + xy[1] ** 2 <= 1 + 1e-15


def test_lens_ray_equals_the_restatement(exe):
    lines = _run(exe, "ray").splitlines()
    assert len(lines) == 64
    for l in lines:
        v = [float(x) for x in l.split()]
        c, n = lens_ref.parse_camera(v)
        sx, sy, u1, u2 = v[n:n + 4]
        o, d = lens_ref.lens_ray(c, sx, sy, u1, u2)
        assert np.allclose(v[n + 4:n + 7], o, rtol=0, atol=1e-12), (v[n + 4:n + 7], o)
        assert np.allclose(v[n + 7:n + 10], d, rtol=0, atol=1e-12), (v[n + 7:n + 10], d)


def test_projection_from_the_lens_equals_the_restatement(exe):
    lines = _run(exe, "proj").splitlines()
    clipped = 0
    for l in lines:
        v = [float(x) for x in l.split()]
        c, n = lens_ref.parse_camera(v)
        p0, p1, (u1, u2), ok = v[n:n + 3], v[n + 3:n + 6], v[n + 6:n + 8], int(v[n + 8])
        ref = lens_ref.project_from_lens(c, p0, p1, u1, u2)
        assert ok == (ref is not None)
        if ref is None:
            continue
        clipped += int(min((c["w2c"] @ np.append(p, 1.0))[2] for p in (p0, p1)) < c["clip_near"])
        q = np.array(v[n + 9:n + 13])
        assert np.allclose(q, np.concatenate(ref), rtol=1e-11, atol=1e-11), (q, ref)
    assert clipped >= 8


def test_lens_adjoints_match_central_differences(exe):
    assert _run(exe, "fd").splitlines()[-1] == "fd ok"


def test_primary_edge_distribution_covers_every_reachable_silhouette(exe):
    out = _run(exe, "dist").splitlines()
    assert out[-1] == "dist ok"
    edges, reachable, pinhole_zero = (int(x) for x in out[-2].split()[1::2])
    # the cases do reach the lens-only ground: edges the pinhole distribution would have dropped
    assert reachable > 300 and pinhole_zero > 50
