"""CPU suite: exact records (rb_exact_record_count, rb_render_exact, rb_exact_round) on the host build of the device headers (tools/cpu_emu).

- Partition sums: the records of the stripes of a 2- and 3-way partition (1- and 4-row stripes), each stripe's gradient descriptor in
  an address order of its own, summed as int64 and rounded once, equal the unpartitioned deterministic render bit for bit in every
  buffer, camera and screen-gradient image included.  One render's records, rounded, equal that render too.
- Crafted records: +inf + +inf = +inf, +inf + -inf = NaN, NaN + x = NaN, carries across three limbs near 2^32, and a zero sum that
  leaves its element untouched.
- Refusals: a wrong count, NULL records, overlapping gradient buffers, and ranks whose record layouts differ.
- dist.render_tiles under deterministic algorithms at world sizes 2 and 3 (gloo) gives every gradient of world size 1 bit for bit.
The same checks on the CUDA library are tests/test_exact_records_gpu.py.

Run as a script (`python tests/test_exact_records_cpu.py <emulator.so> <check>...`) this file is also the subprocess that binds the
emulator in place of the library."""
import ctypes
import os
import socket
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _cases():
    import parity_utils as pu
    small = dict(res=16, spp=4)
    return {
        "glossy_room_both_edges": (dict(pu.CASES["glossy_room_sobol_mb2"], edges=3, **small), "grad"),
        "c2_shadow_blocker_both_edges": (dict(pu.CASES["c2_shadow_blocker_sobol"], edges=3, **small), "grad"),
        "env_ball_sobol_mb2": (dict(pu.CASES["env_ball_sobol_mb2"], **small), "grad"),
        "fisheye_room_primary_edges": (dict(pu.CASES["fisheye_room_primary_edges"], **small), "grad"),
        "distort_room_primary_edges": (dict(pu.CASES["distort_room_primary_edges"], **small), "grad"),
        "gbuffer_bwd_glossy_room": (dict(pu.CASES["gbuffer_bwd_glossy_room"], **small), "grad"),
        "screen_gradient_c1": (dict(pu.SCREEN_CASES["screen_gradient_c1"], **small), "screen"),
    }


CASE_NAMES = ["glossy_room_both_edges", "c2_shadow_blocker_both_edges", "env_ball_sobol_mb2", "fisheye_room_primary_edges", "distort_room_primary_edges",
              "gbuffer_bwd_glossy_room", "screen_gradient_c1"]


def _run(checks):
    from test_device_code_cpu import _build
    so = _build()
    r = subprocess.run([sys.executable, os.path.abspath(__file__), so] + checks, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert [l for l in r.stdout.splitlines() if l.startswith("ok ")] == ["ok " + c for c in checks]


@pytest.mark.parametrize("name", CASE_NAMES)
def test_partition_records_summed_and_rounded_equal_one_deterministic_render(name):
    _run(["partition:" + name])


def test_records_of_one_render_rounded_equal_the_deterministic_render():
    _run(["round_trip"])


def test_crafted_records_sum_non_finite_counts_and_carries():
    _run(["crafted"])


def test_wrong_count_null_records_and_overlapping_buffers_are_refused():
    _run(["refusals"])


# ---------------------------------------------------------------------------------------------------- gloo
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _tile_worker(rank, world, port, emu_so, out_path):
    """One rank of a sharded render under deterministic algorithms, the emulator behind the C ABI."""
    import numpy as np
    import torch
    import torch.distributed as dist
    sys.path.insert(0, HERE)
    from redner_b200 import _lib, dist as rdist
    _lib._lib = _lib._bind(ctypes.CDLL(emu_so))  # this process only
    from redner_b200 import redner as rb
    import parity_utils as pu
    import scenes
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        dev = torch.device("cpu")
        sc = scenes.glossy_room(dev, resolution=(26, 22))
        img = rdist.render_tiles(sc, 4, 2, seed=5, rows_per_stripe=4, sampler_type=rb.SamplerType.sobol, device=dev, backend=rb,
                                 use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
        img.pow(2).sum().backward()
        if rank == 0:
            g = pu.collect_grads(sc)
            np.savez(out_path, image=img.detach().numpy(), **{k: v.numpy() for k, v in g.items()})
    finally:
        dist.destroy_process_group()


def test_gloo_deterministic_render_tiles_is_bitwise_independent_of_world_size(tmp_path):
    import numpy as np
    import torch.multiprocessing as mp
    import test_device_code_cpu as tdc
    emu = tdc._build()
    outs = {}
    for world in (1, 2, 3):
        path = str(tmp_path / ("w%d.npz" % world))
        mp.spawn(_tile_worker, args=(world, _free_port(), emu, path), nprocs=world, join=True)
        outs[world] = dict(np.load(path))
    assert len(outs[1]) > 5 and any(np.count_nonzero(v) for k, v in outs[1].items() if k != "image")
    for world in (2, 3):
        assert set(outs[world]) == set(outs[1]), world
        for k in outs[1]:
            assert outs[world][k].tobytes() == outs[1][k].tobytes(), (world, k)


def _fingerprint_worker(rank, world, port, ret):
    import torch
    import torch.distributed as dist
    from redner_b200 import dist as rdist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rdist.check_records_agree(1000, (1 << 64) - 5, torch.device("cpu"))  # the same on every rank (a fingerprint past 2^63 included)
        try:
            rdist.check_records_agree(1000, 77 + rank, torch.device("cpu"))
            ret[rank] = "not refused"
        except RuntimeError as e:
            ret[rank] = str(e)
    finally:
        dist.destroy_process_group()


def test_ranks_with_different_record_layouts_are_refused():
    import torch.multiprocessing as mp
    ret = mp.Manager().dict()
    mp.spawn(_fingerprint_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    assert all("do not line up" in ret.get(r, "") for r in range(2)), dict(ret)


def main():
    so, names = sys.argv[1], sys.argv[2:]
    sys.path.insert(0, HERE)
    sys.path.insert(0, ROOT)
    import torch
    from redner_b200 import _lib
    _lib._lib = _lib._bind(ctypes.CDLL(so))  # this process only: the emulator exports the same C ABI with host pointers
    from redner_b200 import redner as rb
    import exact_records_check as xc
    dev = torch.device("cpu")
    for name in names:
        if name.startswith("partition:"):
            cfg, kind = _cases()[name.split(":", 1)[1]]
            xc.partition_sums(rb, dev, cfg, kind, (2, 3))
        elif name == "round_trip":
            cfg, kind = _cases()["glossy_room_both_edges"]
            xc.partition_sums(rb, dev, cfg, kind, (1,), rows=(4,))
        elif name == "crafted":
            xc.crafted_records(rb, dev)
        elif name == "refusals":
            xc.refusals(rb, dev)
        print("ok", name, flush=True)


if __name__ == "__main__":
    main()
