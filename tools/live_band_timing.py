"""Cost of running the backward bands over the live samples only, the measurements behind DESIGN.md section 6 "live-pixel bands".

    python tools/live_band_timing.py --parent OTHER_CHECKOUT [--rounds 5] [--workloads c2,c3,c4] [--out result.json]

OTHER_CHECKOUT is a built checkout of another commit (for example the parent of the change), with its library in place.  Each round runs,
one after the other, bench.py --gpus 1 --no-cpu-baseline of both checkouts on C2 (its default steps) and with --steps 3 on C3 and C4, and
this checkout's C2 once more with RB_BAND_BYTES=2^31 (the live samples of C2 in one band).  Per arm the median and min-max of Msamples/s,
the median backward stage times bench.py reports and its kernel launches per step are printed as one JSON line per workload; the band
counts come from one backward pass of each workload on this checkout (rb_scene_last_live_samples), with RB_NO_ZERO_CULL=1 for the count
of a build whose bands cover every sample.  The card's name, power limit and max SM clock are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGES = ("k_backward", "k_bwd_trace", "k_bwd_secondary", "k_bwd_sweep", "k_primary_edge")
ONE_BAND = str(1 << 31)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def bench(tree, workload, env=None):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--no-cpu-baseline", "--workload", workload]
    if workload != "c2":
        cmd += ["--steps", "3"]
    r = subprocess.run(cmd, cwd=tree, capture_output=True, text=True, env=dict(os.environ, **(env or {})))
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError("bench.py failed in %s (%s):\n%s" % (tree, workload, r.stderr[-3000:]))
    out = json.loads(lines[-1])
    k = out["config"]["kernel_ms"]
    return dict(value=out["value"], bwd_ms=out["config"]["bwd_ms"], launches=out["gpu_launches"] // out["steps"] - 1, **{s: k.get(s, 0.0) for s in STAGES})


def bands(workload, env):
    """(live samples, bands) of one backward pass of `workload` on this checkout."""
    probe = ("import json, sys, torch; sys.path[:0] = [%r, %r]; import bench; from redner_b200 import api, redner as rb\n"
             "wl = bench.WORKLOADS[%r]; dev = torch.device('cuda:0')\n"
             "args = api.RenderFunction.serialize_scene(bench.make_scene(wl, dev), wl['spp'], wl['mb'], sampler_type=rb.SamplerType.sobol, device=dev)\n"
             "img = api.RenderFunction.apply(1, *args); img.pow(2).sum().backward(); torch.cuda.synchronize()\n"
             "print(json.dumps(img.grad_fn.c.scene.last_live_samples()))") % (ROOT, os.path.join(ROOT, "tests"), workload)
    r = subprocess.run([sys.executable, "-c", probe], cwd=ROOT, capture_output=True, text=True, env=dict(os.environ, **env))
    if r.returncode != 0:
        raise RuntimeError("band probe failed (%s):\n%s" % (workload, r.stderr[-3000:]))
    return json.loads(r.stdout.strip().splitlines()[-1])


def summary(runs):
    vals = [r["value"] for r in runs]
    med = lambda key: round(statistics.median(r[key] for r in runs), 3)  # noqa: E731
    return dict(msamples_per_s=round(statistics.median(vals), 1), min=round(min(vals), 1), max=round(max(vals), 1), all=[round(v, 1) for v in vals],
                bwd_ms=med("bwd_ms"), launches=runs[-1]["launches"], **{s + "_ms": med(s) for s in STAGES})


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--parent", required=True, help="built checkout of the commit to compare against")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--workloads", default="c2,c3,c4")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    parent = os.path.abspath(a.parent)
    gpu = card()
    arms = {"c2": {"parent": (parent, {}), "this": (ROOT, {}), "this-one-band": (ROOT, {"RB_BAND_BYTES": ONE_BAND})},
            "c3": {"parent": (parent, {}), "this": (ROOT, {})}, "c4": {"parent": (parent, {}), "this": (ROOT, {})}}
    arms = {w: arms[w] for w in a.workloads.split(",")}
    runs = {w: {arm: [] for arm in arms[w]} for w in arms}
    for _ in range(a.rounds):
        for w in arms:
            for arm, (tree, env) in arms[w].items():
                runs[w][arm].append(bench(tree, w, env))
                print(json.dumps(dict(workload=w, arm=arm, **runs[w][arm][-1])), file=sys.stderr, flush=True)
    results = []
    for w in arms:
        r = dict(workload=w, gpu=gpu, rounds=a.rounds, **{arm: summary(runs[w][arm]) for arm in arms[w]})
        live, n = bands(w, {})
        r["live_samples"], r["this"]["bands"] = live, n
        r["parent"]["bands"] = bands(w, {"RB_NO_ZERO_CULL": "1"})[1]
        if "this-one-band" in r:
            r["this-one-band"]["bands"] = bands(w, {"RB_BAND_BYTES": ONE_BAND})[1]
        print(json.dumps(r), flush=True)
        results.append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
