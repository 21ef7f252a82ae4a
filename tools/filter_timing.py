"""Cost of the pixel filters (rb_pixel_filter) on the bench workloads.

    python tools/filter_timing.py [--workloads c2,c3] [--reps 5] [--parent-lib OTHER/libredner_b200.so] [--out result.json]

For each workload of bench.py (same scene, size, samples and bounces, Sobol, both edge samplers, loss = sum(img^2)) the arms
  box          this build, the zero-initialised filter (the 1-pixel box)
  parent-box   --parent-lib: another build of the library (for example the previous commit's), the same call through the same Python
  tent2        this build, a tent of width 2
  gauss3       this build, a Gaussian of width 3
run one after the other, alternating, `reps` times each after one warm-up round.  Per arm the median milliseconds of the forward call
(scene build included: RenderFunction builds its native scene there) and of the backward call (host clock around each, both end in a
synchronisation of the render stream) and the library's own stage times of the last backward pass (rb_scene_last_stage_stats: the
backward bands and the primary-edge pass) are printed as one JSON line per workload, with the card's name and power limit read in the
same run."""
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

FILTERS = {"box": None, "parent-box": None, "tent2": ("tent", 2.0), "gauss3": ("gaussian", 3.0)}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def step(wl, arm, libs):
    """One forward + backward of the workload with the arm's library and filter: (forward ms, backward ms, [bands ms, primary-edge ms])."""
    import bench
    from redner_b200 import _lib, api
    from redner_b200 import redner as rb
    dev = torch.device("cuda:0")
    _lib._lib = libs[arm == "parent-box"]
    try:
        sc = bench.make_scene(wl, dev)
        kw = {} if FILTERS[arm] is None else {"pixel_filter": api.PixelFilter(*FILTERS[arm])}
        args = api.RenderFunction.serialize_scene(sc, wl["spp"], wl["mb"], sampler_type=rb.SamplerType.sobol, device=dev, **kw)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        img = api.RenderFunction.apply(bench.SEED, *args)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        img.pow(2).sum().backward()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        scene = img.grad_fn.c.scene
        stages = (ctypes.c_float * 4)()
        scene._lib.rb_scene_last_stage_stats(scene._handle, stages, None, None)
        return 1e3 * (t1 - t0), 1e3 * (t2 - t1), [stages[1], stages[2]]
    finally:
        _lib._lib = libs[False]


def time_workload(name, reps, arms, libs):
    import bench
    wl = bench.WORKLOADS[name]
    times = {a: [] for a in arms}
    for rep in range(reps + 1):
        for arm in arms:
            r = step(wl, arm, libs)
            if rep > 0:
                times[arm].append(r)
    med = lambda xs: round(statistics.median(xs), 2)  # noqa: E731
    out = dict(workload=name, label=wl["label"], res=wl["res"], spp=wl["spp"], max_bounces=wl["mb"], reps=reps)
    for arm in arms:
        ts = times[arm]
        out[arm] = dict(forward_ms=med([t[0] for t in ts]), backward_ms=med([t[1] for t in ts]), bands_ms=med([t[2][0] for t in ts]),
                        primary_edge_ms=med([t[2][1] for t in ts]), backward_ms_all=[round(t[1], 2) for t in ts])
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workloads", default="c2,c3")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parent-lib", default=None, help="another build of libredner_b200.so to time the box against")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "filter_timing measures on the GPU; there is nothing to measure without one"
    from redner_b200 import _lib
    libs = {False: _lib.load()}
    arms = ["box", "tent2", "gauss3"]
    if a.parent_lib:
        libs[True] = _lib._bind(ctypes.CDLL(os.path.abspath(a.parent_lib)))
        arms = ["parent-box"] + arms
    lines = []
    gpu = card()
    for name in a.workloads.split(","):
        r = time_workload(name, a.reps, arms, libs)
        r["gpu"] = gpu
        print(json.dumps(r), flush=True)
        lines.append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
