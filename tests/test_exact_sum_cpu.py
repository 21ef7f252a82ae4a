"""CPU suite: the exact accumulator of the deterministic backward pass (redner_b200/csrc/rb_exact.cuh), compiled with g++
(tests/exact_sum_check.cpp), against exact rational sums (fractions.Fraction) rounded to nearest-even in float32 and float64.

Covers random lists over the whole float32 exponent range (subnormals included), exact cancellation and exact zeros, halfway ties,
sums beyond FLT_MAX (+-inf), the non-finite rules, carry normalisation at any point, and the same bits for every order of a list.
The device scatter that feeds the same accumulators is tested on the GPU (tests/test_deterministic_gpu.py)."""
import itertools
import math
import os
import random
import shutil
import struct
import subprocess
from fractions import Fraction

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

FLT_MAX = float(np.finfo(np.float32).max)
TINY = 2.0 ** -149  # smallest positive subnormal float32


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.isdir("/usr/local/cuda/include"):
        pytest.skip("needs g++ and the CUDA headers")
    exe = str(tmp_path_factory.mktemp("exact_sum") / "exact_sum_check")
    cmd = ["g++", "-O2", "-std=c++17", "-w", "-include", os.path.join(ROOT, "tools", "cpu_emu", "emu_shim.h"), "-I/usr/local/cuda/include",
           "-I" + os.path.join(ROOT, "include"), os.path.join(HERE, "exact_sum_check.cpp"), "-o", exe]
    subprocess.run(cmd, check=True, timeout=300)
    return exe


def f32_bits(x):
    return struct.unpack("<I", struct.pack("<f", x))[0]


def f64_bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def run(checker, lists, every=0):
    """[(float32 bits, float64 bits)] of the accumulator's sum of each list (python floats that are float32 values)."""
    src = "".join("%d %d %s\n" % (every, len(v), " ".join("%08x" % f32_bits(x) for x in v)) for v in lists)
    out = subprocess.run([checker], input=src, capture_output=True, text=True, check=True, timeout=300).stdout.split()
    return [(int(out[2 * i], 16), int(out[2 * i + 1], 16)) for i in range(len(lists))]


def round_f32(q):
    """Fraction -> float32 value (as a python float), to nearest with ties to even; +-inf beyond the float32 range."""
    if q == 0:
        return 0.0
    sign = -1.0 if q < 0 else 1.0
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()  # 2^e <= a < 2^(e+2)
    if Fraction(2) ** e > a:
        e -= 1
    if Fraction(2) ** (e + 1) <= a:
        e += 1
    quantum = Fraction(2) ** (max(e, -126) - 23)
    m = a / quantum
    n = math.floor(m)
    rem = m - n
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and n % 2 == 1):
        n += 1
    v = n * quantum
    if v >= Fraction(2) ** 128:
        return sign * math.inf
    return sign * float(v)


def expected(values):
    """float32 and float64 bits of the correctly rounded sum, with IEEE's non-finite rules."""
    nan = any(math.isnan(x) for x in values) or (math.inf in values and -math.inf in values)
    if nan:
        return None
    if math.inf in values or -math.inf in values:
        inf = math.inf if math.inf in values else -math.inf
        return f32_bits(inf), f64_bits(inf)
    q = sum((Fraction(x) for x in values), Fraction(0))
    return f32_bits(round_f32(q)), f64_bits(float(q))


def check(checker, lists, every=0):
    got = run(checker, lists, every)
    for v, g in zip(lists, got):
        e = expected(v)
        if e is None:
            assert math.isnan(struct.unpack("<f", struct.pack("<I", g[0]))[0]) and math.isnan(struct.unpack("<d", struct.pack("<Q", g[1]))[0]), v
        else:
            assert g == e, (v, ["%x" % x for x in g], ["%x" % x for x in e])
    return got


def random_float(rng):
    """A float32 from the whole exponent range (subnormals included), either sign."""
    kind = rng.random()
    if kind < 0.15:
        bits = rng.randrange(1, 1 << 23)  # subnormal
    else:
        bits = (rng.randrange(1, 255) << 23) | rng.randrange(0, 1 << 23)
    if rng.random() < 0.5:
        bits |= 1 << 31
    return struct.unpack("<f", struct.pack("<I", bits))[0]


def test_random_lists_over_the_whole_exponent_range(checker):
    rng = random.Random(1)
    lists = [[random_float(rng) for _ in range(rng.randrange(1, 60))] for _ in range(400)]
    # lists of similar magnitude, where the rounding of the sum is not decided by one huge term
    for k in range(200):
        e = rng.randrange(-149, 120)
        lists.append([float(np.float32(rng.uniform(-1, 1) * 2.0 ** e)) for _ in range(rng.randrange(2, 40))])
    check(checker, lists)


def test_cancellation_and_exact_zero(checker):
    got = check(checker, [[1e30, 1.0, -1e30], [1.0, -1.0], [TINY, -TINY], [3.0e38, -3.0e38, 2.0 ** -149], [FLT_MAX, FLT_MAX, -FLT_MAX, -FLT_MAX]])
    assert got[0][0] == f32_bits(1.0)
    assert got[1] == (0, 0) and got[2] == (0, 0)  # an exact zero is +0.0
    assert got[3][0] == 1 and got[4] == (0, 0)


def test_halfway_ties_round_to_even(checker):
    ulp = 2.0 ** -23
    lists = [[1.0, ulp / 2], [1.0 + ulp, ulp / 2], [1.0, ulp / 2, TINY], [1.0, ulp / 2, -TINY], [-1.0, -ulp / 2], [-(1.0 + ulp), -ulp / 2],
             [2.0 ** 24, 1.0], [2.0 ** 24 + 2, 1.0], [2.0 ** -126, 2.0 ** -150 * 2], [16777216.0, 1.0, 1.0]]
    got = check(checker, lists)
    assert got[0][0] == f32_bits(1.0) and got[1][0] == f32_bits(1.0 + 2 * ulp) and got[6][0] == f32_bits(2.0 ** 24)


def test_sums_beyond_the_float_range_round_to_infinity(checker):
    half_ulp_top = 2.0 ** 103
    got = check(checker, [[FLT_MAX, FLT_MAX], [-FLT_MAX, -FLT_MAX], [FLT_MAX, float(np.float32(half_ulp_top))],
                          [FLT_MAX, float(np.float32(half_ulp_top)), -TINY], [FLT_MAX, FLT_MAX, -FLT_MAX]])
    assert got[0][0] == f32_bits(math.inf) and got[1][0] == f32_bits(-math.inf)
    assert got[2][0] == f32_bits(math.inf)      # exactly halfway above FLT_MAX: overflows
    assert got[3][0] == f32_bits(FLT_MAX)       # just below halfway: FLT_MAX
    assert got[4][0] == f32_bits(FLT_MAX)
    assert got[0][1] == f64_bits(2 * FLT_MAX)   # the double result does not overflow


def test_non_finite_rules(checker):
    inf, nan = math.inf, math.nan
    got = run(checker, [[1.0, inf, 2.0], [-inf, 1.0], [inf, inf], [inf, -inf], [nan, 1.0], [inf, nan], [FLT_MAX, FLT_MAX, -inf]])
    as_f32 = [struct.unpack("<f", struct.pack("<I", g[0]))[0] for g in got]
    as_f64 = [struct.unpack("<d", struct.pack("<Q", g[1]))[0] for g in got]
    assert as_f32[0] == inf and as_f32[1] == -inf and as_f32[2] == inf and as_f32[6] == -inf
    assert math.isnan(as_f32[3]) and math.isnan(as_f32[4]) and math.isnan(as_f32[5])
    assert as_f64[0] == inf and as_f64[1] == -inf and math.isnan(as_f64[3]) and math.isnan(as_f64[5])


def test_every_order_and_every_normalisation_gives_the_same_bits(checker):
    rng = random.Random(7)
    base = [[random_float(rng) for _ in range(6)] for _ in range(12)]
    base += [[1e30, 1.0, -1e30, TINY, -3.0, 2.0 ** -130], [FLT_MAX, FLT_MAX, -FLT_MAX, 1.0, -TINY, 5e-39]]
    for v in base:
        perms = [list(p) for p in itertools.permutations(v)]
        results = set(run(checker, perms)) | set(run(checker, perms[:50], every=1)) | set(run(checker, perms[:50], every=3))
        assert len(results) == 1, v
        assert results == {expected(v)}, v
