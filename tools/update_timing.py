"""Host wall time per optimisation step with a new native scene per step (RenderFunction.apply) against one scene updated in place
(api.SceneRenderer / rb_scene_update).

    python tools/update_timing.py [--steps K] [--only NAME ...]
    python tools/update_timing.py --light-scan [--steps K]

For every workload, at 4 spp and at its BASELINE spp, the two paths alternate twice (create, update, create, update).  Each run, in a
process of its own, takes one
warm-up step and K timed steps of: move the parameters, forward, backward of sum(img^2), torch.cuda.synchronize().  Reported per path:
the median step, and the median of the build / update call alone (RenderFunction._unpack, timed on its own after the steps).  Prints one
JSON line per run, then a table of the smaller of the two runs' medians; the first line names the card and its power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import scenes  # noqa: E402
from redner_b200 import api  # noqa: E402


def _bump(t, d):
    with torch.no_grad():
        t.add_(d)


# name: (scene factory, resolution, max_bounces, BASELINE spp, step(scene, k) that moves the parameters)
def _c2_step(sc, k):
    _bump(sc.shapes[1].vertices, 1e-3 * (-1) ** k)


def _teapot_step(sc, k):
    m = sc.materials[-1]
    m.diffuse_reflectance = api.Texture((m.diffuse_reflectance.texels.detach() * (1 + 0.01 * (-1) ** k)).requires_grad_(True))
    sc.camera.position = (sc.camera.position.detach() + 1e-3 * (-1) ** k).requires_grad_(True)


def _vertex_step(shape):
    return lambda sc, k: _bump(sc.shapes[shape].vertices, 1e-3 * (-1) ** k)


WORKLOADS = {
    "c2_shadow_blocker": (scenes.shadow_blocker, 512, 1, 64, _c2_step),
    "c3_teapot": (scenes.teapot, 512, 1, 256, _teapot_step),
    "teapot_geometry": (scenes.teapot_geometry, 512, 1, 256, _vertex_step(5)),
    "c4_bunny_box": (scenes.bunny_box_shifted, 1024, 5, 128, _vertex_step(-1)),
    # (untextured floor: the fixture's textured floor builds its mip pyramid, and an autograd graph, once at construction)
    "hires_room": (lambda dev, resolution: scenes.hires_room(dev, resolution=resolution, textured=False), 512, 2, 64, _vertex_step(3)),
}


def run(name, spp, use_renderer, steps, dev):
    make, res, mb, _, move = WORKLOADS[name]
    sc = make(dev, resolution=(res, res))
    kw = dict(device=dev)
    render = api.SceneRenderer(spp, mb, **kw) if use_renderer else None
    step_ms = []
    for k in range(steps + 1):
        move(sc, k)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if render is not None:
            img = render(sc, k)
        else:
            img = api.RenderFunction.apply(k, *api.RenderFunction.serialize_scene(sc, spp, mb, **kw))
        img.pow(2).sum().backward()
        torch.cuda.synchronize()
        if k > 0:
            step_ms.append(1e3 * (time.perf_counter() - t0))
        del img
    build_ms = []
    scene = render._scene if render is not None else None
    for k in range(steps):
        move(sc, k)
        args = api.RenderFunction.serialize_scene(sc, spp, mb, **kw)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        geometry = render._target(args)[0] if render is not None else None  # (what SceneRenderer would do: None builds a new scene)
        c = api.RenderFunction._unpack((k, k), args, scene=scene if geometry is not None else None, geometry_changed=geometry)
        torch.cuda.synchronize()
        build_ms.append(1e3 * (time.perf_counter() - t0))
        del c
    return statistics.median(step_ms), statistics.median(build_ms)


def light_scan(dev, steps):
    """Light step of geometry updates (rb_scene_build_ms "lights": uploads and the kernels of rb_light_build.cu, synchronised) with
    glossy_room's ball made an emissive mesh of T triangles: the per-light scan is one thread adding T doubles in order, twice."""
    for sphere_res in ((12, 24), (45, 90), (90, 180), (180, 360), (360, 720)):
        sc = scenes.glossy_room(dev, resolution=(64, 64), grad=False, textured=False, sphere_res=sphere_res)
        sc.area_lights.append(api.AreaLight(3, torch.tensor([1.0, 1.0, 1.0])))
        args = api.RenderFunction.serialize_scene(sc, 1, 1, device=dev)
        c = api.RenderFunction._unpack((0, 0), args)
        ms = []
        for k in range(steps + 1):
            _bump(sc.shapes[3].vertices, 1e-4 * (-1) ** k)
            c.scene.update(c.camera, c.shapes, c.materials, c.lights, c.envmap, geometry_changed=True)
            if k > 0:
                ms.append(c.scene.build_ms()["lights"])
        print(json.dumps({"emissive_triangles": int(sc.shapes[3].indices.shape[0]), "lights_ms": round(statistics.median(ms), 3)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--only", nargs="*", default=None)
    ap.add_argument("--light-scan", action="store_true", help="only the light step on long emissive meshes")
    ap.add_argument("--one", nargs=3, default=None, help=argparse.SUPPRESS)  # (workload, spp, path): one run, in a process of its own
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    if a.one:
        print(json.dumps(run(a.one[0], int(a.one[1]), a.one[2] == "update", a.steps, dev)))
        return
    card = {"card": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        card["power_limit"] = q.stdout.strip()
    except Exception:
        card["power_limit"] = "unknown"
    print(json.dumps(card), flush=True)
    if a.light_scan:
        light_scan(dev, a.steps)
        return
    rows = []
    for name in a.only or list(WORKLOADS):
        for spp in (4, WORKLOADS[name][3]):
            res = {"create": [], "update": []}
            for _ in range(2):
                for path in ("create", "update"):
                    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--steps", str(a.steps), "--one", name, str(spp), path],
                                       capture_output=True, text=True)
                    if r.returncode != 0:
                        sys.exit("%s %d %s failed:\n%s" % (name, spp, path, r.stderr[-3000:]))
                    step, build = json.loads(r.stdout.strip().splitlines()[-1])
                    res[path].append((step, build))
                    print(json.dumps({"workload": name, "spp": spp, "path": path, "step_ms": round(step, 3), "build_ms": round(build, 3)}), flush=True)
            rows.append((name, spp, [min(r[0] for r in res[p]) for p in ("create", "update")], [min(r[1] for r in res[p]) for p in ("create", "update")]))
    print("\n| workload | spp | step, create (ms) | step, update (ms) | build (ms) | update (ms) |")
    print("|---|---|---|---|---|---|")
    for name, spp, st, bu in rows:
        print("| %s | %d | %.2f | %.2f | %.2f | %.2f |" % (name, spp, st[0], st[1], bu[0], bu[1]))


if __name__ == "__main__":
    main()
