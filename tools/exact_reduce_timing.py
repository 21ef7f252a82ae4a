"""Cost of exchanging exact records instead of gradients (redner.render_exact + redner.round_exact, what dist.render_tiles does under
torch.use_deterministic_algorithms) against the deterministic backward pass of rb_render, on one GPU with partition 1.

    python tools/exact_reduce_timing.py [--workloads c2,c3,c4] [--reps 5] [--out result.json]

For each workload of bench.py (same scene, size, samples and bounces) the forward pass runs once; then, alternating, `reps` times each
after one warm-up of each: (a) the deterministic rb_render backward pass into zeroed gradient buffers, (b) rb_render_exact into zeroed
records followed by rb_exact_round into zeroed buffers.  Host clock around each, which ends in a synchronisation of the render stream
(both calls synchronise it).  Printed per workload as one JSON line: the medians, the split of (b), the record count and bytes
(13 x 8 bytes per record), whether (a) and (b) agree bit for bit, and the card's name, power limit and SM clock read in the same run.
There is no all-reduce in this measurement: it is the cost on one rank of producing and consuming records."""
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
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def time_workload(name, reps):
    import bench
    from redner_b200 import api, _lib
    from redner_b200 import redner as rb
    wl = bench.WORKLOADS[name]
    dev = torch.device("cuda:0")
    sc = bench.make_scene(wl, dev)
    args = api.RenderFunction.serialize_scene(sc, wl["spp"], wl["mb"], sampler_type=rb.SamplerType.sobol, device=dev)
    img = api.RenderFunction.apply(bench.SEED, *args)
    c = img.grad_fn.c  # the unpacked call of this render (RenderFunction keeps its context on the autograd node)
    d_img = torch.ones_like(img)
    d_ptr = api._ptr(rb, d_img)
    opts = api.RenderFunction.backward_options(c)
    c.scene.set_partition(0, 1, 4)
    probe = api.RenderFunction.gradient_buffers(c)
    count, _ = rb.exact_record_count(c.scene, opts, probe.d_scene)
    times = {"render": [], "records": [], "render_exact": [], "round": []}
    same = True
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        for rep in range(reps + 1):
            g = api.RenderFunction.gradient_buffers(c)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rb.render(c.scene, opts, rb.float_ptr(0), d_ptr, g.d_scene, rb.float_ptr(0), rb.float_ptr(0))
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            h = api.RenderFunction.gradient_buffers(c)
            records = torch.zeros((count, _lib.RB_EXACT_RECORD_WORDS), dtype=torch.int64, device=dev)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            rb.render_exact(c.scene, opts, d_ptr, h.d_scene, None, records)
            torch.cuda.synchronize()
            t3 = time.perf_counter()
            rb.round_exact(c.scene, opts, h.d_scene, None, records)
            torch.cuda.synchronize()
            t4 = time.perf_counter()
            if rep > 0:
                times["render"].append(1e3 * (t1 - t0))
                times["records"].append(1e3 * (t4 - t2))
                times["render_exact"].append(1e3 * (t3 - t2))
                times["round"].append(1e3 * (t4 - t3))
            a = [t for t in api.RenderFunction.gradient_outputs(c, g) if isinstance(t, torch.Tensor)]
            b = [t for t in api.RenderFunction.gradient_outputs(c, h) if isinstance(t, torch.Tensor)]
            same = same and all(x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes() for x, y in zip(a, b))
    finally:
        torch.use_deterministic_algorithms(False)
    med = lambda k: round(statistics.median(times[k]), 2)  # noqa: E731
    return dict(workload=name, label=wl["label"], res=wl["res"], spp=wl["spp"], max_bounces=wl["mb"], reps=reps,
                deterministic_render_ms=med("render"), render_exact_plus_round_ms=med("records"), render_exact_ms=med("render_exact"),
                round_ms=med("round"), deterministic_render_ms_all=[round(t, 2) for t in times["render"]],
                render_exact_plus_round_ms_all=[round(t, 2) for t in times["records"]], records=count,
                record_bytes=count * _lib.RB_EXACT_RECORD_WORDS * 8, bitwise_equal=same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c3,c4")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    gpu = card()
    rows = []
    for w in a.workloads.split(","):
        r = time_workload(w, a.reps)
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
