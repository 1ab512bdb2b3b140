"""fit_count (hyperqueue_b200/csrc/hqs_solver.cuh) on the GPU against exact integer division.

fit_count answers "how many tasks of this variant fit into this free vector, at most cap" once per solver step and in
the pack warps.  The u64 version estimates each quotient in fp32 and fixes it up by +-1 in integer arithmetic, with a
real division when a binding quotient reaches 2^20; the u32 ("narrow") version divides by a magic number derived on the
host.  tests/cuda/fit_probe.cu runs the device function on arrays of cases, with the variant records packed by the
library's own host code.  The reference is exact integer arithmetic: the minimum over the requested resources of
free // amount, where a MAX free amount is unbounded and an `All` request fits once on an untouched resource, clamped to
cap.  Cases: quotients around 2^20 and 2^24 (the fix-up and the division fallback), free amounts at the top of the u64
range (n + d > 2^64), the narrow sentinel, and 10^6 random multi-resource vectors per RT and width."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE = os.path.join(ROOT, "tests", "cuda", "libhqs_fitprobe.so")
MAX64 = (1 << 64) - 1
MAX32 = 0xFFFFFFFF
CAPS = (1, 5, 1 << 20, (1 << 32) - 1)
KS = (0, 1, 2, (1 << 20) - 1, 1 << 20, (1 << 20) + 1, (1 << 24) - 1, (1 << 24) + 1)


@pytest.fixture(scope="module")
def probe():
    from hyperqueue_b200 import _lib
    _lib.load_library()                   # the CUDA runtime the probe links against
    if not os.path.exists(PROBE):
        raise FileNotFoundError(f"{PROBE} is missing: run `python __graft_entry__.py`")
    lib = C.CDLL(PROBE)
    vp = C.c_void_p
    lib.hqs_fit_probe.argtypes = [C.c_uint32, C.c_int, C.c_uint32, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, C.c_char_p, C.c_size_t]
    lib.hqs_fit_probe.restype = C.c_int

    def run(rt, narrow, free, amount, allm, unt, cap, gscale=None):
        free = np.ascontiguousarray(free, dtype=np.uint64)
        amount = np.ascontiguousarray(amount, dtype=np.uint64)
        n, R = free.shape
        allm = np.ascontiguousarray(allm, dtype=np.uint32)
        unt = np.ascontiguousarray(unt, dtype=np.uint32)
        cap = np.ascontiguousarray(cap, dtype=np.uint64)
        gs = None if gscale is None else np.ascontiguousarray(gscale, dtype=np.uint64)
        out = np.zeros(n, dtype=np.uint64)
        err = C.create_string_buffer(256)
        p = lambda a: None if a is None else a.ctypes.data_as(vp)  # noqa: E731
        rc = lib.hqs_fit_probe(rt, int(narrow), n, R, p(free), p(amount), p(allm), p(gs), p(unt), p(cap), p(out), err, 256)
        assert rc == 0, err.value.decode()
        return out
    return run


def reference(free, amount, allm, unt, cap, narrow, gscale=None):
    """Exact fit count per case (numpy uint64 floor division is exact integer division)."""
    free = np.asarray(free, dtype=np.uint64)
    amount = np.asarray(amount, dtype=np.uint64)
    n, R = free.shape
    if gscale is not None:
        amount = amount // np.asarray(gscale, dtype=np.uint64)[None, :R]
    bits = np.uint32(1) << np.arange(R, dtype=np.uint32)[None, :]
    is_all = (np.asarray(allm, dtype=np.uint32)[:, None] & bits) != 0
    untouched = (np.asarray(unt, dtype=np.uint32)[:, None] & bits) != 0
    used = is_all | (amount != 0)
    unbounded = free == np.uint64(MAX32 if narrow else MAX64)
    big = np.uint64(MAX64)
    q = np.where(amount != 0, free // np.maximum(amount, np.uint64(1)), big)
    q = np.where(unbounded, big, q)
    q = np.where(is_all, untouched.astype(np.uint64), q)
    q = np.where(used, q, big)
    return np.minimum(np.asarray(cap, dtype=np.uint64), q.min(axis=1))


def _divisors(max_bits):
    ds = set()
    for j in range(max_bits + 1):
        for d in ((1 << j) - 1, 1 << j, (1 << j) + 1, 3 << (j - 1) if j else 0):
            if 1 <= d < (1 << max_bits):
                ds.add(d)
    return sorted(ds)


def _single_resource_cases(rt, ds, numerators, limit):
    """One requested resource per case, in a slot that moves through the RT slots; the other slots unused."""
    frees, amts, caps = [], [], []
    for i, d in enumerate(ds):
        for n in sorted({x for x in numerators(d) if 0 <= x <= limit}):
            for cap in CAPS:
                r = (i + n) % rt
                f = [0] * rt; a = [0] * rt
                f[r] = n; a[r] = d
                frees.append(f); amts.append(a); caps.append(cap)
    m = len(caps)
    return (np.array(frees, dtype=np.uint64), np.array(amts, dtype=np.uint64), np.zeros(m, np.uint32), np.zeros(m, np.uint32),
            np.array(caps, dtype=np.uint64))


def _check(probe, rt, narrow, free, amount, allm, unt, cap, gscale=None):
    got = probe(rt, narrow, free, amount, allm, unt, cap, gscale)
    exp = reference(free, amount, allm, unt, cap, narrow, gscale)
    bad = np.nonzero(got != exp)[0]
    if bad.size:
        i = int(bad[0])
        lines = [f"{bad.size} of {got.size} cases differ (rt={rt}, narrow={narrow}); first: case {i}",
                 f"  free={[int(x) for x in free[i]]}", f"  amount={[int(x) for x in amount[i]]}",
                 f"  all={int(allm[i]):#x} untouched={int(unt[i]):#x} cap={int(cap[i])}",
                 f"  device {int(got[i])}, exact {int(exp[i])}"]
        over = int((got[bad] > exp[bad]).sum())
        lines.append(f"  over-counts: {over}, under-counts: {bad.size - over}")
        pytest.fail("\n".join(lines))


def _u64_numerators(d):
    out = [k * d + e for k in KS for e in range(-2, 3)]
    return out + [MAX64 - 1, MAX64 - 2, (1 << 64) - d, (1 << 64) - d + 1, (1 << 63) - 1, (1 << 63) + 1]


@pytest.mark.parametrize("rt", [4, 8, 16])
def test_u64_quotient_edges_and_top_of_range(probe, rt):
    """n = k d + e around the fix-up and fallback thresholds, and free amounts within d of 2^64 (n + d > 2^64: the
    estimate is 2^64 / d there and q * d does not fit 64 bits)."""
    _check(probe, rt, False, *_single_resource_cases(rt, _divisors(64), _u64_numerators, MAX64 - 1))


def test_u64_top_of_range_example(probe):
    """free = 2^64 - 2, amount = 2^45: 524287 tasks fit, not 524290."""
    free = np.array([[MAX64 - 1, 0, 0, 0]], dtype=np.uint64)
    amount = np.array([[1 << 45, 0, 0, 0]], dtype=np.uint64)
    got = probe(4, False, free, amount, np.zeros(1, np.uint32), np.zeros(1, np.uint32), np.array([(1 << 32) - 1], np.uint64))
    assert int(got[0]) == ((1 << 64) - 2) // (1 << 45) == 524287


@pytest.mark.parametrize("rt", [4, 8, 16])
def test_u32_quotient_edges_and_sentinel(probe, rt):
    """Narrow amounts: every divisor shape up to 2^31 - 1, n in {0, d - 1, d, 2^31 - 1}, k d + e up to 2^32 - 2, and
    0xFFFFFFFF (unbounded)."""
    def nums(d):
        return [0, d - 1, d, (1 << 31) - 1, MAX32, (MAX32 // d) * d, (MAX32 // d) * d - 1] + \
               [k * d + e for k in KS for e in range(-2, 3)]
    _check(probe, rt, True, *_single_resource_cases(rt, _divisors(31), nums, MAX32))


def test_u32_records_scaled_by_gcd(probe):
    """pack_var32 divides by the per-resource gcd: the probe's free values are the scaled free amounts."""
    rng = np.random.default_rng(7)
    n, R = 20000, 4
    gs = np.array([10000, 2500, 1 << 30, 3], dtype=np.uint64)
    amount = rng.integers(1, 5000, size=(n, R)).astype(np.uint64) * gs[None, :]
    amount[rng.random((n, R)) < 0.3] = 0
    amount[amount.sum(1) == 0, 0] = gs[0]
    free = rng.integers(0, 1 << 31, size=(n, R)).astype(np.uint64)
    free[rng.random((n, R)) < 0.05] = MAX32
    cap = rng.choice(np.array(CAPS, dtype=np.uint64), size=n)
    _check(probe, 4, True, free, amount, np.zeros(n, np.uint32), np.zeros(n, np.uint32), cap, gscale=gs)


def _random_cases(rng, n, rt, narrow):
    top = 31 if narrow else 64
    R = rt
    raw = rng.integers(0, 1 << 63, size=(n, R), dtype=np.uint64) << np.uint64(1) | rng.integers(0, 2, size=(n, R), dtype=np.uint64)
    amount = raw >> rng.integers(64 - top, 64, size=(n, R)).astype(np.uint64)
    amount = np.maximum(amount, np.uint64(1))
    if narrow:
        amount = np.minimum(amount, np.uint64((1 << 31) - 1))
    used = rng.random((n, R)) < 0.6
    allm_b = used & (rng.random((n, R)) < 0.04)
    amount = np.where(used & ~allm_b, amount, np.uint64(0))
    amount = np.where(allm_b & (rng.random((n, R)) < 0.5), np.uint64(1), amount)        # `All` with and without an amount
    none = ~used.any(axis=1)
    amount[none, 0] = 1
    limit = MAX32 if narrow else MAX64
    # free = k * d + rem with rem < d and per-slot quotients k close to a log-uniform row quotient < 2^26 (so that any
    # slot can bind and the minimum is not always 0); a third of the remainders sit at 0, 1, d - 2 or d - 1
    d = np.maximum(amount, np.uint64(1))
    krow = rng.integers(0, 1 << 26, size=(n, 1)).astype(np.uint64) >> rng.integers(0, 27, size=(n, 1)).astype(np.uint64)
    k = (krow << rng.integers(0, 2, size=(n, R)).astype(np.uint64)) + rng.integers(0, 3, size=(n, R)).astype(np.uint64)
    rem = (rng.integers(0, 1 << 63, size=(n, R), dtype=np.uint64) << np.uint64(1)) % d
    edge = rng.integers(0, 4, size=(n, R)).astype(np.uint64)
    rem = np.where(rng.random((n, R)) < 0.33, np.where(edge < 2, np.minimum(edge, d - np.uint64(1)), d - np.minimum(d, edge - np.uint64(1))), rem)
    fits = k <= (np.uint64(limit) - rem) // d                    # k * d + rem <= limit
    free = np.where(fits, k * d + rem, np.uint64(limit) - rem)
    topv = np.uint64(limit) - rng.integers(1, 1 << 20, size=(n, R)).astype(np.uint64)   # just below unbounded
    r = rng.random((n, R))
    free = np.where(r < 0.05, np.uint64(limit), np.where(r < 0.10, topv, free))
    bits = (np.uint32(1) << np.arange(R, dtype=np.uint32))[None, :]
    allm = (allm_b.astype(np.uint32) * bits).sum(axis=1).astype(np.uint32)
    unt = ((rng.random((n, R)) < 0.8).astype(np.uint32) * bits).sum(axis=1).astype(np.uint32)
    cap = np.where(rng.random(n) < 0.5, rng.choice(np.array(CAPS, dtype=np.uint64), size=n),
                   rng.integers(1, 1 << 32, size=n).astype(np.uint64))
    return free, amount, allm, unt, cap


@pytest.mark.parametrize("narrow", [False, True], ids=["u64", "u32"])
@pytest.mark.parametrize("rt", [4, 8, 16])
def test_random_multi_resource_vectors(probe, rt, narrow):
    """10^6 random vectors: the min / select combining over the slots, unused slots, `All` entries and MAX."""
    rng = np.random.default_rng(1000 * rt + int(narrow))
    _check(probe, rt, narrow, *_random_cases(rng, 1_000_000, rt, narrow))
