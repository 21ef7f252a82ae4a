"""Cost of the deterministic backward pass (rb_options.deterministic, torch.use_deterministic_algorithms) on the bench workloads.

    python tools/deterministic_timing.py [--workloads c2,c3,c4] [--reps 5] [--out result.json]

For each workload of bench.py (same scene, size, samples and bounces) the forward pass runs once and the backward pass is timed in
the default and the deterministic mode, alternating, `reps` times each after one warm-up of each; the median milliseconds of each mode
(host clock around backward(), which ends in a synchronisation of the render stream) and the bytes of exact accumulators the
deterministic pass took from the backward scratch (as the library reports them, rb_scene_last_exact_bytes) are printed as one JSON
line per workload, with the card's name and power limit read in the same run.

It also counts, on the test scenes of tests/test_deterministic_gpu.py, the gradient elements that differ between two default-mode
runs and between one band and 1 MiB bands (RB_BAND_BYTES): what deterministic mode removes."""
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


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def time_workload(name, reps):
    import bench
    from redner_b200 import api
    from redner_b200 import redner as rb
    wl = bench.WORKLOADS[name]
    dev = torch.device("cuda:0")
    sc = bench.make_scene(wl, dev)
    args = api.RenderFunction.serialize_scene(sc, wl["spp"], wl["mb"], sampler_type=rb.SamplerType.sobol, device=dev)
    img = api.RenderFunction.apply(bench.SEED, *args)
    grad = torch.ones_like(img)
    scene = img.grad_fn.c.scene  # the native scene of this render (RenderFunction keeps its context on the autograd node)
    times = {False: [], True: []}
    exact_bytes = 0
    for rep in range(reps + 1):
        for det in (False, True):
            torch.use_deterministic_algorithms(det, warn_only=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            img.backward(grad, retain_graph=True)
            torch.cuda.synchronize()
            if rep > 0:
                times[det].append(1e3 * (time.perf_counter() - t0))
            if det:
                exact_bytes = scene.last_exact_bytes()
    torch.use_deterministic_algorithms(False)
    return dict(workload=name, label=wl["label"], res=wl["res"], spp=wl["spp"], max_bounces=wl["mb"], reps=reps,
                default_ms=round(statistics.median(times[False]), 2), deterministic_ms=round(statistics.median(times[True]), 2),
                default_ms_all=[round(t, 2) for t in times[False]], deterministic_ms_all=[round(t, 2) for t in times[True]],
                accumulator_bytes=exact_bytes)


def differences():
    """Gradient elements that differ between two runs and between band sizes, per mode, on the repeatability cases."""
    import test_deterministic_gpu as t
    from redner_b200 import redner as rb
    dev = torch.device("cuda:0")
    out = []
    for name in t.REPEAT_CASES:
        row = dict(case=name)
        for det in (False, True):
            torch.use_deterministic_algorithms(det, warn_only=True)
            a, b = t.render(rb, dev, name), t.render(rb, dev, name)
            os.environ["RB_BAND_BYTES"] = str(1 << 20)
            c = t.render(rb, dev, name)
            del os.environ["RB_BAND_BYTES"]
            n = sum(v.numel() for v in a.values())
            tag = "deterministic" if det else "default"
            row[tag + "_run_to_run"] = int(sum(int((a[k].view(-1) != b[k].view(-1)).sum()) for k in a))
            row[tag + "_band_size"] = int(sum(int((a[k].view(-1) != c[k].view(-1)).sum()) for k in a))
            row["elements"] = n
        torch.use_deterministic_algorithms(False)
        out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c3,c4")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-differences", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    gpu = card()
    rows = []
    for w in a.workloads.split(","):
        r = time_workload(w, a.reps)
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)
    if not a.no_differences:
        for r in differences():
            rows.append(r)
            print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
