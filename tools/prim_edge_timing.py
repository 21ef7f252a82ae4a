"""Cost of projecting the primary-edge adjoints once per edge, the measurements behind DESIGN.md section 6 "Primary edges: one
projection per edge".

    python tools/prim_edge_timing.py --parent OTHER_CHECKOUT [--ablation THIRD_CHECKOUT] [--rounds 5] [--rounds-large 2] [--dumps 3]
                                     [--out result.json]

OTHER_CHECKOUT is a built checkout of another commit (for example the parent of the change), with its library in place; THIRD_CHECKOUT, if
given, a built checkout timed as a third arm on C2 only (for example one whose primary-edge pass skips the projection altogether, a bound
on what any change to the projection can gain).  Each round runs bench.py --gpus 1 --no-cpu-baseline of every checkout, one after the
other, on C2 (its default steps); `rounds-large` rounds do the same with --steps 3 on C3 and C4.  Per arm the median and min-max of
Msamples/s and the median stage times bench.py reports are printed as one JSON line per workload.

Then the outputs: `dumps` runs of each of both checkouts with --dump-outputs on C2 and C3 (alternating), and one of each under
torch.use_deterministic_algorithms (rb_options.deterministic).  Per output array the largest relative L2 difference between two runs of
the parent (its run-to-run spread) and between a run of this checkout and one of the parent are printed, and whether the images and the
deterministic outputs are bit-identical.  The card's name, power limit and max SM clock are read in the same run."""
import argparse
import glob
import itertools
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGES = ("k_forward", "k_backward", "k_bwd_trace", "k_bwd_secondary", "k_bwd_sweep", "k_primary_edge")
DETERMINISTIC = ("import runpy, sys, torch; torch.use_deterministic_algorithms(True); sys.argv = sys.argv[1:]; "
                 "runpy.run_path(sys.argv[0], run_name='__main__')")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def bench(tree, workload, extra=(), deterministic=False):
    cmd = [os.path.join(tree, "bench.py"), "--gpus", "1", "--no-cpu-baseline", "--workload", workload] + list(extra)
    if workload != "c2" and "--steps" not in extra:
        cmd += ["--steps", "3"]
    cmd = [sys.executable] + (["-c", DETERMINISTIC] if deterministic else []) + cmd
    r = subprocess.run(cmd, cwd=tree, capture_output=True, text=True)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError("bench.py failed in %s (%s):\n%s" % (tree, workload, r.stderr[-3000:]))
    out = json.loads(lines[-1])
    k = out["config"]["kernel_ms"]
    return dict(value=out["value"], **{s: k.get(s, 0.0) for s in STAGES})


def summary(runs):
    vals = [r["value"] for r in runs]
    return dict(msamples_per_s=round(statistics.median(vals), 1), min=round(min(vals), 1), max=round(max(vals), 1), all=[round(v, 1) for v in vals],
                **{s + "_ms": round(statistics.median(r[s] for r in runs), 3) for s in STAGES})


def rel_l2(a, b):
    a, b = a.astype(np.float64).ravel(), b.astype(np.float64).ravel()
    n = np.linalg.norm(b)
    d = np.linalg.norm(a - b)
    return float(d / n) if n > 0 else (0.0 if d == 0 else float("inf"))


def load_dump(d):
    return {os.path.basename(p)[:-4]: np.load(p) for p in sorted(glob.glob(os.path.join(d, "*.npy")))}


def compare_outputs(parent_runs, this_runs, parent_det, this_det):
    """Per array: parent's run-to-run spread, largest parent-vs-this difference, and the bit-identity checks."""
    r = {"image_bit_identical": all(np.array_equal(t["image"], p["image"]) for t in this_runs for p in parent_runs),
         "deterministic_bit_identical": sorted(parent_det) == sorted(this_det) and all(np.array_equal(parent_det[k], this_det[k]) for k in parent_det),
         "arrays": {}}
    for name in sorted(parent_runs[0]):
        if name == "image":
            continue
        spread = max((rel_l2(a[name], b[name]) for a, b in itertools.combinations(parent_runs, 2)), default=0.0)
        cross = max(rel_l2(t[name], p[name]) for t in this_runs for p in parent_runs)
        if spread > 0 or cross > 0:
            r["arrays"][name] = dict(parent_spread=float("%.3g" % spread), this_vs_parent=float("%.3g" % cross))
    return r


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--parent", required=True, help="built checkout of the commit to compare against")
    ap.add_argument("--ablation", default=None, help="built checkout timed as a third arm on C2")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--rounds-large", type=int, default=2)
    ap.add_argument("--dumps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    trees = {"parent": os.path.abspath(a.parent), "this": ROOT}
    gpu = card()
    results = []
    for w, rounds in (("c2", a.rounds), ("c3", a.rounds_large), ("c4", a.rounds_large)):
        arms = dict(trees, **({"ablation": os.path.abspath(a.ablation)} if a.ablation and w == "c2" else {}))
        runs = {arm: [] for arm in arms}
        for _ in range(rounds):
            for arm, tree in arms.items():
                runs[arm].append(bench(tree, w))
                print(json.dumps(dict(workload=w, arm=arm, **runs[arm][-1])), file=sys.stderr, flush=True)
        if rounds:
            r = dict(workload=w, gpu=gpu, rounds=rounds, **{arm: summary(runs[arm]) for arm in arms})
            print(json.dumps(r), flush=True)
            results.append(r)
    if a.dumps:
        with tempfile.TemporaryDirectory() as tmp:
            for w in ("c2", "c3"):
                dumps = {arm: [] for arm in trees}
                for k in range(a.dumps):
                    for arm, tree in trees.items():
                        d = os.path.join(tmp, "%s_%s_%d" % (w, arm, k))
                        bench(tree, w, ["--steps", "1", "--warmup", "1", "--dump-outputs", d])
                        dumps[arm].append(load_dump(d))
                det = {}
                for arm, tree in trees.items():
                    d = os.path.join(tmp, "%s_%s_det" % (w, arm))
                    bench(tree, w, ["--steps", "1", "--warmup", "1", "--dump-outputs", d], deterministic=True)
                    det[arm] = load_dump(d)
                r = dict(workload=w, gpu=gpu, outputs=compare_outputs(dumps["parent"], dumps["this"], det["parent"], det["this"]))
                print(json.dumps(r), flush=True)
                results.append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
