"""Cost of the GGX specular lobe (rb_material::specular_model), the measurements behind DESIGN.md section 6 "GGX specular lobe".

    python tools/ggx_timing.py [--reps 5] [--parent-lib OTHER/libredner_b200.so] [--seeds 16] [--out result.json]

1. The teapot (bench workload c3: same scene, size, samples and bounces, Sobol, both edge samplers, loss = sum(img^2)) three ways:
     bp-lean     Blinn-Phong, the kernels rb_render picks (the lean set)
     bp-general  Blinn-Phong with RB_NO_LEAN=1 (the general set)
     ggx         every specular material GGX (the general set)
2. The environment-map scene of the suite (env_ball, 512 x 512, 64 spp, 2 bounces, Blinn-Phong; the general kernels) with this build
   and, with --parent-lib, another build of the library (for example the previous commit's), through the same Python.
   Arms run one after the other, alternating, `reps` times each after one warm-up round; per arm the median milliseconds of the forward
   call (scene build included) and of the backward call (host clock, both end in a synchronisation) and the library's stage times of
   the last backward pass (rb_scene_last_stage_stats / rb_scene_last_backward_stats) are printed as one JSON line per workload.
3. The cost of proposing secondary edges for GGX with the Blinn-Phong LTC table: the glossy room (256 x 256, 16 spp, 2 bounces, primary
   edges off, so that the ball's vertex gradient is all boundary terms of secondary edges) over `seeds` seeds, Blinn-Phong and GGX at the
   same roughness values.  Per lobe: the mean of the x gradient summed over the ball's vertices, its standard error over the seeds, and
   the per-seed backward time.
The card's name and power limit are read in the same run."""
import argparse
import ctypes
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


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def set_model(sc, model):
    for m in sc.materials:
        if m.compute_specular_lighting:
            m.specular_model = model
    return sc


def step(make, spp, mb, lib, no_lean, **kw):
    """One forward + backward: (forward ms, backward ms, [bands, primary edges, trace, secondary, sweep] ms)."""
    from redner_b200 import _lib, api
    from redner_b200 import redner as rb
    dev = torch.device("cuda:0")
    keep = _lib._lib
    _lib._lib = lib
    if no_lean:
        os.environ["RB_NO_LEAN"] = "1"
    try:
        sc = make(dev)
        args = api.RenderFunction.serialize_scene(sc, spp, mb, sampler_type=rb.SamplerType.sobol, device=dev, **kw)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        img = api.RenderFunction.apply(1, *args)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        img.pow(2).sum().backward()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        scene = img.grad_fn.c.scene
        stages, bwd = (ctypes.c_float * 4)(), (ctypes.c_float * 3)()
        scene._lib.rb_scene_last_stage_stats(scene._handle, stages, None, None)
        scene._lib.rb_scene_last_backward_stats(scene._handle, bwd)
        return 1e3 * (t1 - t0), 1e3 * (t2 - t1), [stages[1], stages[2], bwd[0], bwd[1], bwd[2]]
    finally:
        _lib._lib = keep
        os.environ.pop("RB_NO_LEAN", None)


def time_arms(label, arms, spp, mb, reps, **kw):
    """arms: name -> (make, lib, no_lean)."""
    times = {a: [] for a in arms}
    for rep in range(reps + 1):
        for a, (make, lib, no_lean) in arms.items():
            r = step(make, spp, mb, lib, no_lean, **kw)
            if rep > 0:
                times[a].append(r)
    med = lambda xs: round(statistics.median(xs), 2)  # noqa: E731
    out = dict(workload=label, spp=spp, max_bounces=mb, reps=reps)
    for a, ts in times.items():
        out[a] = dict(forward_ms=med([t[0] for t in ts]), backward_ms=med([t[1] for t in ts]), bands_ms=med([t[2][0] for t in ts]),
                      primary_edge_ms=med([t[2][1] for t in ts]), trace_ms=med([t[2][2] for t in ts]), secondary_ms=med([t[2][3] for t in ts]),
                      sweep_ms=med([t[2][4] for t in ts]), backward_ms_all=[round(t[1], 2) for t in ts])
    return out


def secondary_edge_noise(seeds, res=256, spp=16, mb=2):
    import scenes
    from redner_b200 import api
    from redner_b200 import redner as rb
    dev = torch.device("cuda:0")
    out = dict(workload="glossy room, ball vertex x gradient from secondary edges", res=res, spp=spp, max_bounces=mb, seeds=seeds)
    for model in ("blinn_phong", "ggx"):
        g, ms = [], []
        for s in range(seeds):
            sc = set_model(scenes.glossy_room(dev, resolution=(res, res), textured=False), model)
            args = api.RenderFunction.serialize_scene(sc, spp, mb, sampler_type=rb.SamplerType.independent, device=dev,
                                                      use_primary_edge_sampling=False, use_secondary_edge_sampling=True)
            img = api.RenderFunction.apply(100 + s, *args)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            img.pow(2).sum().backward()
            torch.cuda.synchronize()
            ms.append(1e3 * (time.perf_counter() - t0))
            g.append(float(sc.shapes[3].vertices.grad[:, 0].sum()))
        mean = statistics.mean(g)
        se = statistics.stdev(g) / len(g) ** 0.5
        out[model] = dict(mean=mean, std_err=se, rel_std_err=se / abs(mean) if mean else None, backward_ms=round(statistics.median(ms), 2))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seeds", type=int, default=16)
    ap.add_argument("--parent-lib", default=None, help="another build of libredner_b200.so to time the environment-map scene against")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "ggx_timing measures on the GPU; there is nothing to measure without one"
    import bench
    import scenes
    from redner_b200 import _lib
    lib = _lib.load()
    gpu = card()
    wl = bench.WORKLOADS["c3"]

    def teapot(model):
        return lambda dev: set_model(bench.make_scene(wl, dev), model)
    results = [time_arms(wl["label"], {"bp-lean": (teapot("blinn_phong"), lib, False), "bp-general": (teapot("blinn_phong"), lib, True),
                                       "ggx": (teapot("ggx"), lib, False)}, wl["spp"], wl["mb"], a.reps)]
    env = {"this": (lambda dev: scenes.env_ball(dev, resolution=(512, 512)), lib, False)}
    if a.parent_lib:
        env["parent"] = (env["this"][0], _lib._bind(ctypes.CDLL(os.path.abspath(a.parent_lib))), False)
    results.append(time_arms("env_ball 512x512 (general kernels)", env, 64, 2, a.reps, use_secondary_edge_sampling=False))
    results.append(secondary_edge_noise(a.seeds))
    for r in results:
        r["gpu"] = gpu
        print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
