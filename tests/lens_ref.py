"""Float64 restatement of the thin-lens camera (DESIGN.md "thin-lens camera"), written from its definition and independent of the device
headers: the concentric disc map, the lens ray and the projection from a lens point.  Used by tests/test_lens_functions_cpu.py."""
import math

import numpy as np


def concentric(u1, u2):
    """Shirley-Chiu's concentric map of [0, 1)^2 onto the unit disc."""
    a, b = 2 * u1 - 1, 2 * u2 - 1
    if a == 0 and b == 0:
        return 0.0, 0.0
    if a * a > b * b:
        r, phi = a, (math.pi / 4) * (b / a)
    else:
        r, phi = b, math.pi / 2 - (math.pi / 4) * (a / b)
    return r * math.cos(phi), r * math.sin(phi)


def parse_camera(v):
    """The camera as lens_functions prints it; returns (dict, number of values read)."""
    c = dict(width=int(v[0]), height=int(v[1]), r=v[2], f=v[3])
    c["c2w"] = np.array(v[4:20]).reshape(4, 4)
    c["w2c"] = np.array(v[20:36]).reshape(4, 4)
    c["intr_inv"] = np.array(v[36:45]).reshape(3, 3)
    c["intr"] = np.array(v[45:54]).reshape(3, 3)
    c["clip_near"] = v[54]
    return c, 55


def lens_ray(c, sx, sy, u1, u2):
    """(origin, direction) in world space of film position (sx, sy) through the lens sample (u1, u2)."""
    aspect = c["width"] / c["height"]
    d = c["intr_inv"] @ np.array([(sx - 0.5) * 2, (sy - 0.5) * -2 / aspect, 1.0])
    L = np.array([*(c["r"] * np.array(concentric(u1, u2))), 0.0])
    F = d * (c["f"] / d[2])
    n = (F - L) / np.linalg.norm(F - L)
    o = c["c2w"] @ np.append(L, 1.0)
    w = c["c2w"][:3, :3] @ n
    return o[:3] / o[3], w / np.linalg.norm(w)


def project_from_lens(c, p0, p1, u1, u2):
    """Screen positions of the ends of world-space segment (p0, p1) seen from lens sample (u1, u2), after the camera-space near clip, or
    None when both ends lie behind the near plane."""
    def cam(p):
        q = c["w2c"] @ np.append(np.asarray(p, float), 1.0)
        return q[:3] / q[3]
    a, b, cn = cam(p0), cam(p1), c["clip_near"]
    if a[2] < cn and b[2] < cn:
        return None
    if a[2] < cn:
        a = b + (cn - b[2]) / (a[2] - b[2]) * (a - b)
    elif b[2] < cn:
        b = a + (cn - a[2]) / (b[2] - a[2]) * (b - a)
    lx, ly = (c["r"] * np.array(concentric(u1, u2)))
    f, aspect = c["f"], c["width"] / c["height"]

    def screen(P):
        Q = np.array([lx / f + (P[0] - lx) / P[2], ly / f + (P[1] - ly) / P[2], 1.0])
        ip = c["intr"] @ Q
        return np.array([(ip[0] / ip[2] + 1) * 0.5, (-(ip[1] / ip[2]) * aspect + 1) * 0.5])
    return screen(a), screen(b)
