"""CPU suite: the GGX specular lobe (rb_material::specular_model == RB_SPECULAR_GGX, DESIGN.md section "GGX").

Function level, on tests/ggx_functions.cpp (the device headers compiled for the host with Real = double):
- eval, pdf and sample against the float64 restatement below, written from the definition: alpha from 1e-3 to 1, incidence from the
  normal to grazing, two-sided materials seen from below, and frames perturbed by a normal map;
- the spec pdf integrates to 1 over the sphere of reflected directions (quadrature) and to at most 1 over the directions a sample keeps;
- 10^6 samples per case fall into bins as the pdf says: chi-square over bins with at least 5 expected samples, p > 1e-4 per case;
- d_bsdf_eval's GGX branch against central differences for kd, ks, roughness, the shading normal, the normal-map texel, wi and wo, at
  the reference's tolerance (1e-3, relative where the derivative exceeds 1).
Scene level, on the host emulator (tools/cpu_emu):
- an explicit "blinn_phong" renders the default bit for bit (images and gradients); an update that changes only specular_model equals
  a new scene; an out-of-range specular_model is refused with a message naming the field;
- on the glossy room with GGX materials, gradients of a fixed weighted loss agree with finite differences (fd_check of the pixel-filter
  suite) for a roughness, a specular reflectance and the position of the ball, whose shadow and reflection edges are secondary edges;
- with torch.use_deterministic_algorithms(True) a GGX render is bitwise repeatable and independent of the band size, and a gloo
  render_tiles at world size 2 equals world size 1.

Run as a script (`python tests/test_ggx_cpu.py <emulator.so> <check>...`) this file is also the subprocess that binds the emulator in place
of the library; tests/test_ggx_gpu.py calls the same checks on the GPU."""
import ctypes
import math
import os
import shutil
import socket
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)


# ---------------------------------------------------------------------------------------------------- the lobe, restated in float64
def _lum(c):
    return 0.212671 * c[0] + 0.715160 * c[1] + 0.072169 * c[2]


def _lambda(a2, n, v):
    c = np.dot(n, v)
    tan2 = (1.0 - c * c) / (c * c)
    return (-1.0 + math.sqrt(1.0 + a2 * tan2)) / 2.0


def _ndf(a2, n, h):
    c = np.dot(n, h)
    return a2 / (math.pi * (c * c * (a2 - 1.0) + 1.0) ** 2)


def _lobe_normal(two_sided, fn, wi):
    return -fn if two_sided and np.dot(wi, fn) < 0 else fn


def ref_eval(rough, two_sided, kd, ks, fn, gn, wi, wo):
    """f |cos wo| = kd |n.wo| / pi + F D G2 / (4 |n.wi|) with the guards of the Blinn-Phong BSDF (min_rough = 0)."""
    gi, go = np.dot(gn, wi), np.dot(gn, wo)
    sh_wi, sh_wo = abs(np.dot(fn, wi)), abs(np.dot(fn, wo))
    if gi * go < 0 or (not two_sided and gi < 0 and go < 0) or sh_wi == 0 or sh_wo <= 1e-3 or abs(go) <= 1e-3:
        return np.zeros(3)
    a2 = max(rough, 1e-6)
    out = kd * sh_wo / math.pi
    n = _lobe_normal(two_sided, fn, wi)
    h = (wi + wo) / np.linalg.norm(wi + wo)
    if np.dot(n, wi) > 0 and np.dot(n, h) > 0:
        G2 = 1.0 / (1.0 + _lambda(a2, n, wi) + _lambda(a2, n, wo))
        F = ks + (1.0 - ks) * max(1.0 - abs(np.dot(h, wo)), 0.0) ** 5
        out = out + F * _ndf(a2, n, h) * G2 / (4.0 * sh_wi)
    return out


def ref_pdf(rough, two_sided, kd, ks, fn, gn, wi, wo):
    gi, go = np.dot(gn, wi), np.dot(gn, wo)
    if gi * go < 0 or (not two_sided and gi < 0 and go < 0):
        return 0.0
    wd, ws = _lum(kd), _lum(ks)
    pd, ps = (wd / (wd + ws), ws / (wd + ws)) if wd + ws > 0 else (0.5, 0.5)
    pdf = pd * abs(np.dot(fn, wo)) / math.pi
    n = _lobe_normal(two_sided, fn, wi)
    h = (wi + wo) / np.linalg.norm(wi + wo)
    if ps > 0 and np.dot(n, wi) > 0 and np.dot(n, h) > 0:
        a2 = max(rough, 1e-6)
        pdf += ps * _ndf(a2, n, h) / (1.0 + _lambda(a2, n, wi)) / (4.0 * np.dot(n, wi))
    return pdf


def ref_sample_spec(rough, two_sided, fx, fy, fn, gn, wi, u1, u2):
    """The specular branch of bsdf_sample_dir: visible normals by spherical caps (Dupuy & Benyoub 2023) in the frame, mirrored when a
    two-sided material is seen from below; a zero vector when the sample fails."""
    gi = np.dot(gn, wi)
    if not two_sided and gi < 0:
        return np.zeros(3)
    alpha = math.sqrt(max(rough, 1e-6))
    wl = np.array([np.dot(wi, fx), np.dot(wi, fy), np.dot(wi, fn)])
    s = -1.0 if two_sided and wl[2] < 0 else 1.0
    wl[2] *= s
    if wl[2] <= 0:
        return np.zeros(3)
    vs = np.array([alpha * wl[0], alpha * wl[1], wl[2]])
    vs /= np.linalg.norm(vs)
    phi = 2 * math.pi * u1
    z = (1 - u2) * (1 + vs[2]) - vs[2]
    st = math.sqrt(max(1 - z * z, 0.0))
    hs = np.array([st * math.cos(phi), st * math.sin(phi), z]) + vs
    hl = np.array([alpha * hs[0], alpha * hs[1], hs[2]])
    hl /= np.linalg.norm(hl)
    h = fx * hl[0] + fy * hl[1] + fn * (s * hl[2])
    d = 2 * np.dot(wi, h) * h - wi
    return np.zeros(3) if np.dot(gn, d) * gi < 0 else d


# ---------------------------------------------------------------------------------------------------- function level
@pytest.fixture(scope="module")
def functions(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.isdir("/usr/local/cuda/include"):
        pytest.skip("needs g++ and the CUDA headers")
    exe = str(tmp_path_factory.mktemp("ggx") / "ggx_functions")
    cmd = ["g++", "-O2", "-std=c++17", "-w", "-DRB_REAL_DOUBLE", "-include", os.path.join(ROOT, "tools", "cpu_emu", "emu_shim.h"), "-I/usr/local/cuda/include",
           "-I" + os.path.join(ROOT, "include"), '-DRB_DATA_DIR="%s"' % os.path.join(ROOT, "redner_b200", "data"), os.path.join(HERE, "ggx_functions.cpp"),
           "-o", exe, "-lpthread"]
    subprocess.run(cmd, check=True, timeout=900)

    def run(mode):
        r = subprocess.run([exe, mode], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        return r.stdout.strip().splitlines()
    return run


def test_eval_pdf_sample_match_the_restatement(functions):
    lines = functions("grid")
    assert len(lines) == 5 * 4 * 4 * 6
    spec_seen = sampled = 0
    for line in lines:
        v = [float(x) for x in line.split()[1:]]
        rough, two_sided = v[0], bool(v[1])
        kd, ks = np.array(v[2:5]), np.array(v[5:8])
        fx, fy, fn, gn, wi, wo = (np.array(v[8 + 3 * k:11 + 3 * k]) for k in range(6))
        f, pdf, u1, u2, w_sel, ws = np.array(v[26:29]), v[29], v[30], v[31], v[32], np.array(v[33:36])
        ef = ref_eval(rough, two_sided, kd, ks, fn, gn, wi, wo)
        assert np.allclose(f, ef, rtol=1e-7, atol=1e-12), (line, ef)
        ep = ref_pdf(rough, two_sided, kd, ks, fn, gn, wi, wo)
        assert math.isclose(pdf, ep, rel_tol=1e-7, abs_tol=1e-12), (line, ep)
        assert w_sel > _lum(kd) / (_lum(kd) + _lum(ks))
        es = ref_sample_spec(rough, two_sided, fx, fy, fn, gn, wi, u1, u2)
        assert np.allclose(ws, es, rtol=1e-7, atol=1e-9), (line, es)
        spec_seen += np.any(ef - kd * abs(np.dot(fn, wo)) / math.pi > 1e-6 * np.abs(ef).max(initial=1e-30))
        sampled += bool(np.any(ws))
    assert spec_seen > 100 and sampled > 100, (spec_seen, sampled)  # (the lobe is exercised, not only its guards)


def test_spec_pdf_integrates_to_one(functions):
    for line in functions("quad"):
        _, alpha, theta, variant, total, kept = line.split()
        # quadrature on 4000 x 512 points around the mirror direction; the grazing alpha = 0.02 case is the hardest (2e-3)
        assert abs(float(total) - 1.0) < 5e-3, line
        assert float(kept) <= float(total) + 1e-9, line


def test_sample_histogram_matches_the_pdf(functions):
    from scipy.stats import chi2
    lines = functions("hist")
    assert len(lines) == 18
    for line in lines:
        v = line.split()
        counts = np.array([float(x) for x in v[4:]]).reshape(-1, 2)
        obs, exp = counts[:, 0], counts[:, 1]
        assert abs(obs.sum() - 1e6) < 0.5 and abs(exp.sum() - 1e6) < 1e6 * 5e-3, line[:80]
        big = exp >= 5
        o = np.append(obs[big], obs[~big].sum())
        e = np.append(exp[big], exp[~big].sum())
        e *= o.sum() / e.sum()
        keep = e > 0
        if keep.sum() == 1:  # (seen from below a one-sided surface every sample fails, as the pdf says)
            assert np.all(o[keep] == 1e6) and abs(e[keep][0] - 1e6) < 1e-6 * 1e6, line[:80]
            continue
        stat = float((((o - e) ** 2)[keep] / e[keep]).sum())
        p = chi2.sf(stat, int(keep.sum()) - 1)
        assert p > 1e-4, (v[1:4], stat, int(keep.sum()), p)


def test_adjoint_matches_finite_differences(functions):
    lines = functions("fd")
    assert lines[-1].startswith("fd checks") and int(lines[-1].split()[2]) >= 2000


# ---------------------------------------------------------------------------------------------------- scene level (shared with the GPU suite)
def ggx_room(dev, res, textured=True, models=("ggx",)):
    """The glossy room with `models` on its specular materials (floor, ball), in that order."""
    import scenes
    sc = scenes.glossy_room(dev, resolution=(res, res), textured=textured)
    spec = [m for m in sc.materials if m.compute_specular_lighting]
    for m, model in zip(spec, list(models) * len(spec)):
        m.specular_model = model
    return sc


def render(rb, dev, sc, spp, seed, mb=2, backward=True, **kw):
    """Image and gradients (of sum(W * img), W the pixel-filter suite's weight image) of one RenderFunction call."""
    import parity_utils as pu
    from redner_b200 import api
    from test_pixel_filter_cpu import weight_image
    kw.setdefault("sampler_type", rb.SamplerType.sobol)
    args = api.RenderFunction.serialize_scene(sc, spp, mb, device=dev, backend=rb, **kw)
    img = api.RenderFunction.apply(seed, *args)
    if backward:
        (weight_image(img.shape).to(img.device) * img).sum().backward()
    return img.detach().cpu().numpy(), pu.collect_grads(sc)


def assert_same(a, b, what):
    (ia, ga), (ib, gb) = a, b
    assert ia.tobytes() == ib.tobytes(), what
    assert ga.keys() == gb.keys() and ga, what
    for k in ga:
        assert ga[k].numpy().tobytes() == gb[k].numpy().tobytes(), (what, k)


def explicit_default_check(rb, dev, res=12, spp=2):
    """specular_model="blinn_phong" given explicitly == the default, bit for bit; GGX renders something else."""
    import scenes
    base = render(rb, dev, scenes.glossy_room(dev, resolution=(res, res)), spp, 3)
    assert_same(base, render(rb, dev, ggx_room(dev, res, models=("blinn_phong",)), spp, 3), "explicit blinn_phong")
    assert render(rb, dev, ggx_room(dev, res), spp, 3)[0].tobytes() != base[0].tobytes()


def update_check(rb, dev, res=12, spp=2):
    """A Scene.update that changes only specular_model renders what a new scene renders (both ways)."""
    import torch
    from test_pixel_filter_cpu import native_scene

    def image(c):
        img = torch.zeros(res, res, 3)
        rb.render(c.scene, c.options, rb.float_ptr(img.data_ptr()), rb.float_ptr(0), None, rb.float_ptr(0), rb.float_ptr(0))
        return img.numpy().tobytes()
    for first, second in ((("blinn_phong",), ("ggx",)), (("ggx",), ("blinn_phong",)), (("ggx", "blinn_phong"), ("blinn_phong", "ggx"))):
        c = native_scene(rb, dev, ggx_room(dev, res, models=first), None)
        new = native_scene(rb, dev, ggx_room(dev, res, models=second), None)
        c.scene.update(new.camera, new.shapes, new.materials, new.lights, None, geometry_changed=False)
        assert image(c) == image(new), (first, second)


def refusals_check(rb, dev):
    """Out-of-range models are refused, by api.Material and by rb_scene_create / rb_scene_update, with a message naming the field."""
    from redner_b200 import api
    from test_pixel_filter_cpu import native_scene
    with pytest.raises(ValueError, match="specular_model"):
        api.Material(specular_model="phong")
    c = native_scene(rb, dev, ggx_room(dev, 8), None)
    for bad in (2, -1):
        mats = [rb.Material(*m_args(rb, m), specular_model=bad) for m in c.materials]
        with pytest.raises(RuntimeError, match="specular_model"):
            rb.Scene(c.camera, c.shapes, mats, c.lights, None, c.scene.use_gpu, c.scene.gpu_index, True, True)
        with pytest.raises(RuntimeError, match="specular_model"):
            c.scene.update(c.camera, c.shapes, mats, c.lights, None, geometry_changed=False)


def m_args(rb, m):
    """redner.Material arguments that rebuild the native material `m` (its textures and flags)."""
    t = m._c
    tex = []
    for name, cls in (("diffuse_reflectance", rb.Texture3), ("specular_reflectance", rb.Texture3), ("roughness", rb.Texture1),
                      ("generic_texture", rb.TextureN), ("normal_map", rb.Texture3)):
        w = cls.__new__(cls)
        w._c = getattr(t, name)
        tex.append(w)
    return tex + [t.compute_specular_lighting, t.two_sided, t.use_vertex_color]


def fd_checks(rb, dev, res, spp, fd_spp, seeds):
    """Gradients of the GGX glossy room against central finite differences (fd_check): the ball's roughness and specular reflectance,
    and the ball's position along x (its silhouette is a primary edge, its shadow and its reflection on the floor are secondary edges)."""
    import torch
    from redner_b200 import api
    from test_pixel_filter_cpu import fd_check

    def make():
        return ggx_room(dev, res, textured=False)

    def ball(sc):
        return next(m for m in sc.materials if m.compute_specular_lighting and m.roughness.texels.numel() == 1 and m is not sc.materials[0])

    def set_tex(attr):
        def move(sc, d):
            m = ball(sc)
            t = getattr(m, attr)
            setattr(m, attr, api.Texture((t.texels.detach() + d).requires_grad_(True), t.uv_scale))
        return move, lambda sc: float(getattr(ball(sc), attr).texels.grad.sum())

    def ball_shape(sc):
        mid = sc.materials.index(ball(sc))
        return next(s for s in sc.shapes if s.material_id == mid)

    def shift(sc, d):
        s = ball_shape(sc)
        with torch.no_grad():
            s.vertices[:, 0] += d
    out = {}
    for name, (move, grad_of) in (("roughness", set_tex("roughness")), ("specular", set_tex("specular_reflectance"))):
        out[name] = fd_check(rb, dev, make, move, grad_of, None, spp, fd_spp, seeds, 0.02, mb=2)
    out["ball_x"] = fd_check(rb, dev, make, shift, lambda sc: float(ball_shape(sc).vertices.grad[:, 0].sum()), None, spp, fd_spp, seeds, 0.05, mb=2)

    return out


# The render that tests/test_ggx_gpu.py compares between the GPU and the emulator.
COMPARE = dict(res=24, spp=8, seed=9, mb=2)


def compare_render(rb, dev):
    """Image and gradients of the GGX glossy room at COMPARE, Sobol, both edge samplers, as numpy arrays."""
    img, g = render(rb, dev, ggx_room(dev, COMPARE["res"]), COMPARE["spp"], COMPARE["seed"], mb=COMPARE["mb"], use_secondary_edge_sampling=True)
    return dict(image=img, **{k: v.numpy() for k, v in g.items()})


def deterministic_check(rb, dev, res=12, spp=2):
    """Deterministic mode: a GGX render is bitwise repeatable and independent of the band size (RB_BAND_BYTES: many small bands on the GPU)."""
    import torch
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        a = render(rb, dev, ggx_room(dev, res), spp, 5)
        assert_same(a, render(rb, dev, ggx_room(dev, res), spp, 5), "repeat")
        os.environ["RB_BAND_BYTES"] = str(1 << 20)
        try:
            assert_same(a, render(rb, dev, ggx_room(dev, res), spp, 5), "band size")
        finally:
            del os.environ["RB_BAND_BYTES"]
    finally:
        torch.use_deterministic_algorithms(False)


# ---------------------------------------------------------------------------------------------------- on the emulator
def _run(checks, timeout=2400):
    from test_device_code_cpu import _build
    so = _build()
    r = subprocess.run([sys.executable, os.path.abspath(__file__), so] + checks, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert [l for l in r.stdout.splitlines() if l.startswith("ok ")] == ["ok " + c for c in checks]


def test_explicit_blinn_phong_is_the_default_bit_for_bit():
    _run(["explicit_default"])


def test_specular_model_update_equals_a_new_scene():
    _run(["update"])


def test_out_of_range_specular_model_is_refused():
    _run(["refusals"])


def test_ggx_gradients_match_finite_differences():
    _run(["fd"])


def test_ggx_deterministic_repeatable_and_band_independent():
    _run(["deterministic"])


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _tile_worker(rank, world, port, emu_so, out_path):
    """One rank of a sharded GGX render under deterministic algorithms, the emulator behind the C ABI."""
    import torch
    import torch.distributed as dist
    sys.path.insert(0, HERE)
    from redner_b200 import _lib, dist as rdist
    _lib._lib = _lib._bind(ctypes.CDLL(emu_so))  # this process only
    from redner_b200 import redner as rb
    import parity_utils as pu
    from test_pixel_filter_cpu import weight_image
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        dev = torch.device("cpu")
        sc = ggx_room(dev, 14)
        img = rdist.render_tiles(sc, 2, 2, seed=5, rows_per_stripe=4, sampler_type=rb.SamplerType.sobol, device=dev, backend=rb,
                                 use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
        (weight_image(img.shape) * img).sum().backward()
        if rank == 0:
            g = pu.collect_grads(sc)
            np.savez(out_path, image=img.detach().numpy(), **{k: v.numpy() for k, v in g.items()})
    finally:
        dist.destroy_process_group()


def test_gloo_render_tiles_with_ggx_is_independent_of_world_size(tmp_path):
    import torch.multiprocessing as mp
    import test_device_code_cpu as tdc
    emu = tdc._build()
    outs = {}
    for world in (1, 2):
        path = str(tmp_path / ("w%d.npz" % world))
        mp.spawn(_tile_worker, args=(world, _free_port(), emu, path), nprocs=world, join=True)
        outs[world] = dict(np.load(path))
    assert len(outs[1]) > 5 and any(np.count_nonzero(v) for k, v in outs[1].items() if k != "image")
    assert set(outs[2]) == set(outs[1])
    for k in outs[1]:
        assert outs[2][k].tobytes() == outs[1][k].tobytes(), k


def main():
    so, names = sys.argv[1], sys.argv[2:]
    sys.path.insert(0, ROOT)
    import torch
    from redner_b200 import _lib
    _lib._lib = _lib._bind(ctypes.CDLL(so))  # this process only: the emulator exports the same C ABI with host pointers
    from redner_b200 import redner as rb
    dev = torch.device("cpu")
    for name in names:
        if name == "explicit_default":
            explicit_default_check(rb, dev)
        elif name == "update":
            update_check(rb, dev)
        elif name == "refusals":
            refusals_check(rb, dev)
        elif name == "fd":
            fd_checks(rb, dev, 16, 32, 256, 4)
        elif name == "deterministic":
            deterministic_check(rb, dev)
        elif name.startswith("compare:"):
            np.savez(name[len("compare:"):], **compare_render(rb, dev))
        print("ok", name, flush=True)


if __name__ == "__main__":
    main()
