"""The FP64 path's arithmetic claims, checked against exact integers (README, "The central idea").

The product headers' primitives (ntt_fp_body.cuh, modarith.cuh) are compiled for the host by tests/fp_exact with the
emulation build's floating-point flags, and every result is compared with Python integers:
  * it is an integer-valued double equal to the exact value of its rounding form (the quotient is rint of the stated
    floating-point expression; the remainder is then computed exactly), congruent to the exact result mod p;
  * its magnitude is within the bound the bookkeeping uses: fp_prod_bound for products, fp_renormed_bound after
    renormalisation, [0, p) after fp_to_canonical, [0, 2q) for the lazy Shoup product.
Operands come in structured classes: extremes, the stage bounds of the transform schedules, and operands on the rounding
boundaries, where the quotient estimate lands within a few ulps of a half-integer.

The renorm masks the library computes are re-derived here from the stated bounds for the generic schedule and the statically
scheduled kernels', and the generic FP64 transform, run with each schedule's pass list and masks on worst-case inputs, must
give the reference's words without any pass writing a value beyond the bookkeeping's bound.

Device coverage: on the device DMUL, DFMA, DADD and cvt.rni are IEEE round-to-nearest as on the host, so these checks carry
over; the device-only bit tricks of fp_to_canonical and fp_from_u64 are covered by the GPU parity tests only."""
import ctypes as C
import os
import subprocess
from collections import defaultdict

import numpy as np
import pytest

from params import PARAMS

HERE = os.path.dirname(os.path.abspath(__file__))
LIMIT = 2.0 ** 53
N_PER_WIDTH = 1_000_000  # operand tuples per primitive per prime width
STATIC_SCHED = {12: [4, 4, 4], 13: [3, 3, 3, 4], 14: [3, 3, 4, 4]}  # the statically scheduled kernels' (NttSched)
COUNTS = defaultdict(lambda: defaultdict(int))  # primitive -> prime width -> operand tuples checked

dp = C.POINTER(C.c_double)
up = C.POINTER(C.c_uint64)
i64 = C.c_longlong


@pytest.fixture(scope="session")
def fpx():
    subprocess.run(["make", "-C", os.path.join(HERE, "fp_exact")], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
    L = C.CDLL(os.path.join(HERE, "fp_exact", "_build", "libfp_exact.so"))
    L.fpx_mulmod.argtypes = [C.c_int, i64, dp, dp, dp, C.c_double, dp]
    L.fpx_mulmod2.argtypes = [i64, dp, dp, C.c_double, C.c_double, dp]
    L.fpx_renorm.argtypes = [C.c_int, i64, dp, C.c_double, C.c_double, dp]
    L.fpx_to_canonical.argtypes = [C.c_int, i64, dp, C.c_double, C.c_double, up]
    L.fpx_prod_bound.argtypes = [i64, C.c_double, dp, dp]
    L.fpx_renormed_bound.argtypes = [C.c_double]
    L.fpx_renormed_bound.restype = C.c_double
    L.fpx_inner.argtypes = [i64, C.c_int, dp, dp, dp, C.c_double, C.c_double, dp, dp, up]
    L.fpx_ntt.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_double, dp, dp, C.c_double, C.c_double,
                          C.c_uint, C.c_uint, up, i64, dp]
    L.fpx_ntt.restype = i64
    L.fpx_shoup.argtypes = [C.c_int, i64, up, up, up, C.c_uint64, up]
    L.fpx_barrett64.argtypes = [i64, up, C.c_uint64, C.c_uint64, up]
    L.fpx_barrett128.argtypes = [i64, up, up, C.c_uint64, C.c_uint64, C.c_uint64, up]
    L.fpx_addsub.argtypes = [C.c_int, i64, up, up, C.c_uint64, up]
    return L


def ptr(a, t=dp):
    return a.ctypes.data_as(t)


def obj(a):
    """exact Python integers of an integer-valued float64 / int64 / uint64 array"""
    if a.dtype == np.float64:
        a = a.astype(np.int64)
    return a.astype(object)


# ------------------------------------------------------------------------------------------------------------------
# primes and their schedules
# ------------------------------------------------------------------------------------------------------------------
def is_prime(v):
    if v < 2:
        return False
    for sp in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        if v % sp == 0:
            return v == sp
    d, s = v - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for a in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        x = pow(a, d, v)
        if x in (1, v - 1):
            continue
        for _ in range(s - 1):
            x = x * x % v
            if x == v - 1:
                break
        else:
            return False
    return True


def largest_ntt_prime(bits, n):
    """the largest prime = 1 mod 2n below 2^bits"""
    v = ((1 << bits) - 1) // (2 * n) * (2 * n) + 1
    while not is_prime(v):
        v -= 2 * n
    return v


@pytest.fixture(scope="session")
def contexts(emu_lib):
    """name -> (n, emulation context) for every parameter set"""
    from sunscreen_b200.lib import B200Context
    return {name: (n, B200Context(n, moduli, t, lib=emu_lib)) for name, (n, moduli, t) in PARAMS.items()}


def device_primes(ctx):
    """the context's device primes in index order (key primes, auxiliary primes, then t when batching)"""
    out, f, i = [], C.c_uint(), C.c_uint()
    while True:
        p = C.c_uint64()
        ctx.L.lib.b200_debug_fp_masks(ctx.h, len(out), 0, C.byref(p), C.byref(f), C.byref(i))
        if not p.value:
            return out
        out.append(p.value)


@pytest.fixture(scope="session")
def primes_by_width(contexts):
    """every FP64-path prime (<= 49 bits) of tests/params.py, the auxiliary primes the contexts pick and the largest 49-bit
    NTT-friendly primes for n = 4096 ... 32768, and (for the integer primitives) every wider one, grouped by width"""
    ps = set()
    for name, (n, ctx) in contexts.items():
        ps.update(device_primes(ctx))
        for lv in range(ctx.levels):
            ps.update(ctx.level_info(lv)["bsk"])
    ps.update(largest_ntt_prime(49, n) for n in (4096, 8192, 16384, 32768))
    ps = {p for p in ps if is_prime(p) and p > 2}
    by = defaultdict(list)
    for p in sorted(ps):
        by[p.bit_length()].append(p)
    return dict(by)


def fp_widths(by):
    return {w: ps for w, ps in by.items() if w <= 49}


def generic_schedule(logn):
    """ntt_body.cuh ntt_schedule: stages per forward pass"""
    rem = logn
    a = 1 if rem >= 4 else 0
    while a <= rem // 4 and (rem - 4 * a) % 3:
        a += 1
    if a > rem // 4:
        out, r = [], rem
        while r > 0:
            L = 4 if r >= 4 and r not in (5, 6) else (3 if r >= 3 else r)
            out.append(L)
            r -= L
        return sorted(out)
    while rem - 4 * (a + 3) >= 0 and (rem - 4 * (a + 3)) % 3 == 0:
        a += 3
    return [3] * ((rem - 4 * a) // 3) + [4] * a


def prod_bound(p, y):
    """b200_bfv.cu / ntt_fp_body.cuh: the magnitude of a product of an input |y| <= 2^53"""
    return p * (0.5 + 3.0 * y / LIMIT) + 1.0


def pass_bounds(p, L, fwd_mask, inv_mask):
    """the bookkeeping re-derived: per pass (execution order) the bound on what it writes, for the given masks; a bound above
    2^53 (inf) marks a pass whose values could overflow"""
    p = float(p)
    renormed = 0.76 * p
    fwd, b = [], p
    for pi, stages in enumerate(L):
        if fwd_mask >> pi & 1:
            b = renormed
        for _ in range(stages):
            b += prod_bound(p, b)
            b = b if b <= LIMIT else float("inf")
        fwd.append(b)
    inv, b = [], p
    for step, stages in enumerate(reversed(L)):
        if inv_mask >> step & 1:
            b = renormed
        for _ in range(stages):
            b = float("inf") if 2.0 * b > LIMIT else max(2.0 * b, prod_bound(p, 2.0 * b))
        inv.append(b)
    return fwd, inv


def derive_masks(p, L):
    """renormalise a pass's inputs exactly when the pass could otherwise exceed 2^53"""
    fwd = inv = 0
    for pi in range(len(L)):
        if pass_bounds(p, L, fwd, 0)[0][pi] == float("inf"):
            fwd |= 1 << pi
    for step in range(len(L)):
        if pass_bounds(p, L, 0, inv)[1][step] == float("inf"):
            inv |= 1 << step
    assert all(b <= LIMIT for b in sum(pass_bounds(p, L, fwd, inv), [])), (p, L)
    return fwd, inv


def stage_bounds(p):
    """every intermediate bound the bookkeeping produces for the schedules in use (as integers)"""
    out = set()
    for logn in range(10, 16):
        for L in [generic_schedule(logn)] + ([STATIC_SCHED[logn]] if logn in STATIC_SCHED else []):
            fm, im = derive_masks(p, L)
            b = float(p)
            for pi, stages in enumerate(L):
                b = 0.76 * p if fm >> pi & 1 else b
                for _ in range(stages):
                    b += prod_bound(p, b)
                    out.add(int(b))
            b = float(p)
            for step, stages in enumerate(reversed(L)):
                b = 0.76 * p if im >> step & 1 else b
                for _ in range(stages):
                    out.update((int(2 * b), int(prod_bound(p, 2 * b))))
                    b = max(2.0 * b, prod_bound(p, 2.0 * b))
    return sorted(v for v in out if v <= 2 ** 53)


# ------------------------------------------------------------------------------------------------------------------
# exact models of the rounding forms
# ------------------------------------------------------------------------------------------------------------------
def rint_exact(y, d):
    """round-half-even of the exact product y * d (y: integers, d: float64 array), as the magic-number form computes it
    (one rounding of the exact fma result)"""
    mant, ex = np.frexp(d)
    M = obj((mant * 2.0 ** 53).astype(np.int64))
    s = (53 - ex).astype(np.int64)
    num = y * M
    us, at = np.unique(s, return_inverse=True)
    half = np.array([1 << int(v - 1) for v in us], dtype=object)[at]
    q = (num + half) >> s.astype(object)
    tie = (num & (2 * half - 1)) == half
    q = np.where(tie & (q % 2 == 1), q - 1, q)
    return np.where(M == 0, 0, q)


def check_remainder(label, p, prod, r, q, bound=None):
    """r (float64) is the integer prod - q p, congruent to prod mod p, and |r| <= bound"""
    assert np.all(np.isfinite(r)) and np.all(r == np.rint(r)), (label, p, "non-integer result")
    assert np.all(np.abs(r) <= LIMIT), (label, p)
    ro = obj(r)
    want = prod - q * p
    bad = np.nonzero(ro != want)[0]
    assert bad.size == 0, (label, p, "result != exact value of the rounding form", bad[:5], ro[bad[:5]], want[bad[:5]])
    assert np.all((prod - ro) % p == 0), (label, p, "not congruent")
    if bound is not None:
        bad = np.nonzero(np.abs(r) > bound)[0]
        assert bad.size == 0, (label, p, "magnitude above the stated bound", r[bad[:5]], bound[bad[:5]])


def split(total, parts):
    return [total // parts + (1 if i < total % parts else 0) for i in range(parts)]


# ------------------------------------------------------------------------------------------------------------------
# operand classes
# ------------------------------------------------------------------------------------------------------------------
def special_w(p):
    return [0, 1, p - 1, (p - 1) // 2, (p + 1) // 2]


def mul_operands(p, count, ylim, rng):
    """(y, w) pairs, |y| <= ylim, 0 <= w < p: extremes x special twiddles, stage bounds, rounding-boundary operands (the y
    nearest to (m + 1/2) p / w and its neighbours +-1, +-2) and uniform draws"""
    sy = {0, 1, p - 1, 2 ** 52, 2 ** 53} | set(stage_bounds(p))
    sy = sorted({s * sg for s in sy for sg in (1, -1) if s <= ylim})
    sw = special_w(p)
    ys, ws = [], []
    # extremes x special twiddles, extremes x random twiddles
    for y in sy:
        for w in sw:
            ys.append(y)
            ws.append(w)
    rw = rng.integers(1, p, size=64)
    for y in sy:
        ys.extend([y] * len(rw))
        ws.extend(rw.tolist())
    y0 = np.array(ys, dtype=np.int64)
    w0 = np.array(ws, dtype=np.int64)
    rest = max(count - y0.size, 10_000)
    nb = rest * 3 // 4 // 5
    # rounding boundaries: twiddles random or special, m across the whole range and at its ends
    wb = rng.integers(1, p, size=nb)
    wb[: nb // 8] = rng.choice(np.array(sw[1:], dtype=np.int64), size=nb // 8)
    wbo = obj(wb)
    mmax = (ylim * wbo) // p - 1
    frac = rng.random(nb)
    m = np.array([int(f * int(mm)) for f, mm in zip(frac, mmax)], dtype=object)
    m[: nb // 8] = mmax[: nb // 8] - np.arange(nb // 8)
    m = np.where(rng.random(nb) < 0.5, -m - 1, m)
    yb = ((2 * m + 1) * p + wbo) // (2 * wbo)
    yb = np.concatenate([yb + d for d in (-2, -1, 0, 1, 2)])
    wb = np.tile(wb, 5)
    yb = np.array([min(max(int(v), -ylim), ylim) for v in yb], dtype=np.int64)
    nu = rest - yb.size
    yu = rng.integers(-ylim, ylim + 1, size=nu, dtype=np.int64)
    wu = rng.integers(0, p, size=nu, dtype=np.int64)
    return np.concatenate([y0, yb, yu]), np.concatenate([w0, wb, wu])


def renorm_operands(p, count, rng):
    """x with |x| <= 2^53: extremes, x = (m + 1/2) p + delta for m near +-2^53 / p and across the range, uniform draws"""
    sx = {0, 1, p - 1, p, p + 1, 2 ** 52, 2 ** 53 - 1, 2 ** 53} | set(stage_bounds(p))
    x0 = np.array(sorted({s * sg for s in sx for sg in (1, -1)}), dtype=np.int64)
    rest = max(count - x0.size, 10_000)
    nb = rest * 3 // 4 // 5
    mmax = 2 ** 53 // p - 1
    m = rng.integers(0, mmax + 1, size=nb, dtype=np.int64)
    m[: nb // 4] = mmax - rng.integers(0, min(mmax, 1000) + 1, size=nb // 4)
    m = np.where(rng.random(nb) < 0.5, -m - 1, m)
    xb = ((2 * obj(m) + 1) * p) // 2
    xb = np.concatenate([xb + d for d in (-2, -1, 0, 1, 2)])
    xb = np.array([min(max(int(v), -2 ** 53), 2 ** 53) for v in xb], dtype=np.int64)
    xu = rng.integers(-2 ** 53, 2 ** 53 + 1, size=rest - xb.size, dtype=np.int64)
    return np.concatenate([x0, xb, xu])


# ------------------------------------------------------------------------------------------------------------------
# the FP64 primitives
# ------------------------------------------------------------------------------------------------------------------
def per_prime(by, rng_seed):
    for width, ps in sorted(fp_widths(by).items()):
        for p, cnt in zip(ps, split(N_PER_WIDTH, len(ps))):
            yield width, p, cnt, np.random.default_rng(rng_seed + p)


def bounds_of(fpx, p, y):
    out = np.empty(y.size)
    fpx.fpx_prod_bound(y.size, float(p), ptr(y), ptr(out))
    return out


def test_fp_mulmod_forms(fpx, primes_by_width):
    """fp_mulmod (magic-number quotient, exact for |y w/p| < 2^51: the BEHZ kernels pass |y| < 2^49), fp_mulmod_x (XU
    quotient, any |y| <= 2^53) and fp_mulmod_term of both parities"""
    for width, p, cnt, rng in per_prime(primes_by_width, 1):
        pd = float(p)
        for ylim, kinds in ((2 ** 51, (0, 2)), (2 ** 53, (1, 3))):
            y, w = mul_operands(p, cnt, ylim, rng)
            yd, wd = y.astype(np.float64), w.astype(np.float64)
            wp = wd / pd
            prod = obj(y) * obj(w)
            q = rint_exact(obj(y), wp) if kinds[0] == 0 else obj(np.rint(yd * wp))
            bound = bounds_of(fpx, p, yd)
            for kind in kinds:
                out = np.empty(y.size)
                fpx.fpx_mulmod(kind, y.size, ptr(yd), ptr(wd), ptr(wp), pd, ptr(out))
                label = ["fp_mulmod", "fp_mulmod_x", "fp_mulmod_term(even)", "fp_mulmod_term(odd)"][kind]
                check_remainder(label, p, prod, out, q, bound)
                COUNTS[label][width] += y.size


def test_fp_mulmod2(fpx, primes_by_width):
    """fp_mulmod2 over the range its call sites give it: lazy |a| up to 2^53 (the transform's butterflies) times b < p"""
    for width, p, cnt, rng in per_prime(primes_by_width, 2):
        pd = float(p)
        a, b = mul_operands(p, cnt, 2 ** 53, rng)
        ad, bd = a.astype(np.float64), b.astype(np.float64)
        q = obj(np.rint((ad * bd) * (1.0 / pd)))
        out = np.empty(a.size)
        fpx.fpx_mulmod2(a.size, ptr(ad), ptr(bd), pd, 1.0 / pd, ptr(out))
        check_remainder("fp_mulmod2", p, obj(a) * obj(b), out, q, bounds_of(fpx, p, ad))
        # the bound itself is the formula the bookkeeping states
        assert np.array_equal(bounds_of(fpx, p, ad), prod_bound(pd, np.abs(ad)))
        COUNTS["fp_mulmod2"][width] += a.size


def test_fp_renorm_and_canonical(fpx, primes_by_width):
    """fp_renorm / fp_renorm_x: |x - q p| <= 0.76 p for |x| <= 2^53; fp_to_canonical<false/true>: x mod p exactly"""
    for width, p, cnt, rng in per_prime(primes_by_width, 3):
        pd, pinv = float(p), 1.0 / float(p)
        x = renorm_operands(p, cnt, rng)
        xd = x.astype(np.float64)
        xo = obj(x)
        renormed = fpx.fpx_renormed_bound(pd)
        assert renormed == 0.76 * pd
        for xu, q in ((0, rint_exact(xo, np.full(x.size, pinv))), (1, obj(np.rint(xd * pinv)))):
            out = np.empty(x.size)
            fpx.fpx_renorm(xu, x.size, ptr(xd), pd, pinv, ptr(out))
            label = ["fp_renorm", "fp_renorm_x"][xu]
            check_remainder(label, p, xo, out, q, np.full(x.size, renormed))
            COUNTS[label][width] += x.size
            canon = np.empty(x.size, dtype=np.uint64)
            fpx.fpx_to_canonical(xu, x.size, ptr(xd), pd, pinv, ptr(canon, up))
            bad = np.nonzero(obj(canon) != xo % p)[0]
            assert bad.size == 0, ("fp_to_canonical", xu, p, x[bad[:5]], canon[bad[:5]])
            COUNTS[f"fp_to_canonical<{'true' if xu else 'false'}>"][width] += x.size


@pytest.mark.parametrize("K", list(range(1, 17)))
def test_inner_product_extremes(fpx, primes_by_width, K):
    """inner products of K = 1 ... 16 terms as the BEHZ kernels form them, every term at its positive or negative extreme
    (y w = (p -+ 1) / 2 mod p) for inputs y < 2^49: each partial sum stays an exact integer <= 2^53 and the final
    fp_renorm / fp_to_canonical are exact.  Covers 16 residues against 49-bit auxiliary primes (n16384_49_16x24)."""
    for width, ps in sorted(fp_widths(primes_by_width).items()):
        for p in ps[-2:]:
            rng = np.random.default_rng(p + K)
            cnt = 2000
            pd = float(p)
            y = rng.integers(1, min(2 ** 49, 2 ** 62), size=(cnt, K), dtype=np.int64)
            y[y % p == 0] = 1
            sign = rng.random((cnt, K)) < 0.5
            sign[: cnt // 4] = True
            sign[cnt // 4: cnt // 2] = False
            target = np.where(sign, (p - 1) // 2, (p + 1) // 2).astype(object)
            yo = obj(y)
            w = np.array([t * pow(int(v) % p, -1, p) % p for t, v in zip(target.ravel(), yo.ravel())], dtype=np.int64)
            w = w.reshape(cnt, K)
            yd, wd = y.astype(np.float64), w.astype(np.float64)
            wp = wd / pd
            partial = np.empty((cnt, K))
            renormed = np.empty(cnt)
            canon = np.empty(cnt, dtype=np.uint64)
            fpx.fpx_inner(cnt, K, ptr(yd), ptr(wd), ptr(wp), pd, 1.0 / pd, ptr(partial), ptr(renormed), ptr(canon, up))
            # exact terms: the first with the magic-number quotient, then alternating parities
            terms = np.empty((cnt, K), dtype=object)
            for i in range(K):
                q = rint_exact(yo[:, i], wp[:, i]) if i == 0 or (i - 1) % 2 == 0 else obj(np.rint(yd[:, i] * wp[:, i]))
                terms[:, i] = yo[:, i] * obj(w[:, i]) - q * p
            exact = np.cumsum(terms, axis=1)
            assert np.all(np.abs(partial) <= LIMIT), (p, K)
            assert np.all(obj(partial) == exact), (p, K, "a partial sum is not exact")
            total = exact[:, -1]
            assert np.all(obj(canon) == total % p), (p, K)
            assert np.all((obj(renormed) - total) % p == 0) and np.all(np.abs(renormed) <= 0.76 * pd), (p, K)
            COUNTS["inner product (K terms)"][width] += cnt * K


# ------------------------------------------------------------------------------------------------------------------
# the integer primitives (modarith.cuh)
# ------------------------------------------------------------------------------------------------------------------
def int_operands(q, count, rng, top):
    """values in [0, top): extremes, neighbours of multiples of q, uniform draws"""
    sv = sorted({v % top for v in (0, 1, q - 1, q, q + 1, 2 * q - 1, 2 * q, 4 * q - 1, top - 1, top - 2, (q - 1) // 2,
                                   (q + 1) // 2)})
    nb = count // 3
    k = rng.integers(0, max(1, min(top // q, 2 ** 62)), size=nb, dtype=np.int64).astype(object)
    d = rng.integers(-2, 3, size=nb).astype(object)
    vb = [(int(a) * q + int(b)) % top for a, b in zip(k, d)]
    vu = rng.integers(0, top, size=count - nb - len(sv), dtype=np.uint64)
    return np.concatenate([np.array(sv + vb, dtype=np.uint64), vu])


def per_int_prime(by, seed):
    for width, ps in sorted(by.items()):
        for p, cnt in zip(ps, split(N_PER_WIDTH, len(ps))):
            yield width, p, cnt, np.random.default_rng(seed + p)


def test_shoup(fpx, primes_by_width):
    """shoup_mul_lazy: any 64-bit y times w < q, result in [0, 2q) and congruent; shoup_mul: canonical"""
    for width, q, cnt, rng in per_int_prime(primes_by_width, 4):
        y = int_operands(q, cnt, rng, 2 ** 64)
        w = int_operands(q, cnt, rng, q)
        rng.shuffle(w)
        wq = np.array([(int(v) << 64) // q for v in w], dtype=np.uint64)
        exact = obj(y) * obj(w) % q
        for lazy in (1, 0):
            out = np.empty(y.size, dtype=np.uint64)
            fpx.fpx_shoup(lazy, y.size, ptr(y, up), ptr(w, up), ptr(wq, up), q, ptr(out, up))
            oo = obj(out)
            if lazy:
                assert np.all(oo < 2 * q) and np.all(oo % q == exact), ("shoup_mul_lazy", q)
            else:
                assert np.all(oo == exact), ("shoup_mul", q)
            COUNTS["shoup_mul_lazy" if lazy else "shoup_mul"][width] += y.size


def test_barrett(fpx, primes_by_width):
    """barrett64 of any 64-bit word; barrett128 of inputs below 2^127: near 2^127, near multiples of q, products of
    canonical values, uniform draws (q up to 61 bits: the reference's auxiliary base)"""
    for width, q, cnt, rng in per_int_prime(primes_by_width, 5):
        x = int_operands(q, cnt, rng, 2 ** 64)
        out = np.empty(x.size, dtype=np.uint64)
        fpx.fpx_barrett64(x.size, ptr(x, up), q, 2 ** 64 // q, ptr(out, up))
        assert np.all(obj(out) == obj(x) % q), ("barrett64", q)
        COUNTS["barrett64"][width] += x.size
        r = (1 << 128) // q
        n4 = cnt // 4
        top = [(1 << 127) - 1 - d for d in range(64)]
        k = rng.integers(0, 2 ** 62, size=n4, dtype=np.int64).astype(object) * ((1 << 127) // q // 2 ** 62)
        near_q = [(int(a) * q + int(d)) % (1 << 127) for a, d in zip(k, rng.integers(-2, 3, size=n4))]
        a = int_operands(q, n4, rng, q)
        b = int_operands(q, n4, rng, q)
        prods = list(obj(a) * obj(b))
        hi = rng.integers(0, 2 ** 63, size=cnt - len(top) - len(near_q) - len(prods), dtype=np.uint64).astype(object)
        uni = list((hi << 64) + rng.integers(0, 2 ** 64, size=hi.size, dtype=np.uint64).astype(object))
        v = np.array(top + near_q + prods + uni, dtype=object)
        lo = np.array([int(t) & (2 ** 64 - 1) for t in v], dtype=np.uint64)
        hi = np.array([int(t) >> 64 for t in v], dtype=np.uint64)
        out = np.empty(v.size, dtype=np.uint64)
        fpx.fpx_barrett128(v.size, ptr(lo, up), ptr(hi, up), q, r & (2 ** 64 - 1), r >> 64, ptr(out, up))
        bad = np.nonzero(obj(out) != v % q)[0]
        assert bad.size == 0, ("barrett128", q, v[bad[:5]])
        COUNTS["barrett128"][width] += v.size


def test_add_sub_neg(fpx, primes_by_width):
    for width, q, cnt, rng in per_int_prime(primes_by_width, 6):
        a = int_operands(q, cnt, rng, q)
        b = int_operands(q, cnt, rng, q)
        rng.shuffle(b)
        ao, bo = obj(a), obj(b)
        for op, name, want in ((0, "add_mod", (ao + bo) % q), (1, "sub_mod", (ao - bo) % q), (2, "neg_mod", (-ao) % q)):
            out = np.empty(a.size, dtype=np.uint64)
            fpx.fpx_addsub(op, a.size, ptr(a, up), ptr(b, up), q, ptr(out, up))
            assert np.all(obj(out) == want), (name, q)
            COUNTS[name][width] += a.size


# ------------------------------------------------------------------------------------------------------------------
# renorm masks and the transform against the schedules that run
# ------------------------------------------------------------------------------------------------------------------
def lib_masks(ctx, idx, schedule):
    p, f, i = C.c_uint64(), C.c_uint(), C.c_uint()
    rc = ctx.L.lib.b200_debug_fp_masks(ctx.h, idx, schedule, C.byref(p), C.byref(f), C.byref(i))
    return (f.value, i.value) if rc == 0 else None


def test_renorm_masks_match_the_bounds(contexts):
    """for every FP64 prime of every parameter set: the masks of the generic schedule and of the statically scheduled
    kernels equal the ones re-derived here from the stated bounds, and the emulation's transforms use the generic ones"""
    checked = 0
    for name, (n, ctx) in contexts.items():
        logn = n.bit_length() - 1
        for idx, p in enumerate(device_primes(ctx)):
            got = [lib_masks(ctx, idx, s) for s in (0, 1, 2)]
            if p.bit_length() > 49 or n >= 32768:  # integer path (the split n = 32768 transform has no FP64 path)
                assert got == [None, None, None], (name, idx, p, got)
                continue
            assert got[1] == derive_masks(p, generic_schedule(logn)), (name, hex(p), got)
            assert got[0] == got[1], (name, hex(p))
            if logn in STATIC_SCHED:
                assert got[2] == derive_masks(p, STATIC_SCHED[logn]), (name, hex(p), got)
            else:
                assert got[2] is None
            checked += 1
    assert checked > 100


def twiddles(p, n):
    """the library's FP64 tables, recomputed from the minimal primitive 2n-th root: fwd[bitrev(i)] = psi^i, inv = fwd^-1"""
    c = (p - 1) // (2 * n)
    g = next(x for x in (pow(a, c, p) for a in range(2, 100000)) if pow(x, n, p) == p - 1)
    g2, cur, psi = g * g % p, g, g
    for _ in range(n):
        psi = min(psi, cur)
        cur = cur * g2 % p
    logn = n.bit_length() - 1
    fwd = [0] * n
    v = 1
    for i in range(n):
        fwd[int(format(i, f"0{logn}b")[::-1], 2)] = v
        v = v * psi % p
    inv = [pow(x, -1, p) for x in fwd]
    return fwd, inv


def exact_ntt(a, fwd, inv, p, forward):
    """the negacyclic transform in exact integers (bit-reversed output), one stage per loop trip"""
    n = a.shape[-1]
    x = a.astype(object).copy()
    if forward:
        m = 1
        while m < n:
            t = n // (2 * m)
            v = x.reshape(-1, m, 2, t)
            w = np.array(fwd[m:2 * m], dtype=object)[None, :, None]
            u, s = v[:, :, 0, :].copy(), v[:, :, 1, :] * w % p
            v[:, :, 0, :], v[:, :, 1, :] = (u + s) % p, (u - s) % p
            m *= 2
    else:
        m = n // 2
        while m >= 1:
            t = n // (2 * m)
            v = x.reshape(-1, m, 2, t)
            w = np.array(inv[m:2 * m], dtype=object)[None, :, None]
            u, s = v[:, :, 0, :].copy(), v[:, :, 1, :].copy()
            v[:, :, 0, :], v[:, :, 1, :] = (u + s) % p, (u - s) * w % p
            m //= 2
        x = x * pow(n, -1, p) % p
    return x.astype(np.uint64)


def worst_inputs(p, n, rng):
    """all p - 1, alternating 0 / p - 1, all (p - 1) / 2 and random words"""
    return np.stack([np.full(n, p - 1), np.tile([0, p - 1], n // 2), np.full(n, (p - 1) // 2),
                     rng.integers(0, p, size=n, dtype=np.int64)]).astype(np.uint64)


@pytest.mark.parametrize("logn", [12, 13, 14])
def test_transform_schedules_at_the_bound(fpx, emu_lib, contexts, logn):
    """the generic FP64 transform driven with the generic and the static pass lists and the masks the library computes
    for them, on the largest 49-bit NTT-friendly prime and the parameter sets' widest FP64 primes of this size: words equal
    the exact transform (and the reference's, where it is built), and no pass writes a value beyond its bound"""
    n = 1 << logn
    ps = {largest_ntt_prime(49, n), largest_ntt_prime(48, n)}
    for name, (nn, ctx) in contexts.items():
        if nn == n:
            ps.update(p for p in device_primes(ctx) if p.bit_length() >= 47 and p.bit_length() <= 49)
    import refseal
    from sunscreen_b200.lib import B200Context
    ref = refseal.RefLib.get() if refseal.have_ref() else None
    for p in sorted(ps):
        fwd, inv = twiddles(p, n)
        # the library's masks for this prime: a context whose first key prime is p
        ctx = B200Context(n, [p, largest_ntt_prime(30, n)], 65537 if n == 4096 else 786433, lib=emu_lib)
        rng = np.random.default_rng(p)
        x = worst_inputs(p, n, rng)
        want_f = exact_ntt(x, fwd, inv, p, True)
        want_i = exact_ntt(x, fwd, inv, p, False)
        if ref is not None:
            assert np.array_equal(ref.ntt_forward(p, x), want_f) and np.array_equal(ref.ntt_inverse(p, x), want_i)
        for schedule, L in ((1, generic_schedule(logn)), (2, STATIC_SCHED[logn])):
            fm, im = lib_masks(ctx, 0, schedule)
            bf, bi = pass_bounds(p, L, fm, im)
            La = (C.c_int * len(L))(*L)
            inv_n = pow(n, -1, p)
            twf, twi = np.array(fwd, dtype=np.float64), np.array(inv, dtype=np.float64)
            for forward, want, bounds in ((1, want_f, bf), (0, want_i, bi)):
                data = x.copy()
                amax = np.zeros(8)
                nonint = fpx.fpx_ntt(forward, logn, len(L), La, float(p), ptr(twf), ptr(twi), float(inv_n), float(inv_n * inv[1] % p), fm, im,
                                     ptr(data, up), data.shape[0], ptr(amax))
                tag = (hex(p), L, "forward" if forward else "inverse", hex(fm), hex(im))
                assert nonint == 0, tag
                assert np.array_equal(data, want), tag
                over = [(s, amax[s], bounds[s]) for s in range(len(L)) if not amax[s] <= bounds[s] <= LIMIT]
                assert not over, (tag, over)
                COUNTS[f"transform logn {logn}"][p.bit_length()] += data.size
        ctx.close()


def test_report_counts(capsys):
    """operand tuples each primitive saw, per prime width (>= 10^6 for every primitive and FP64 width)"""
    if not COUNTS:
        pytest.skip("run with the primitive tests")
    with capsys.disabled():
        print("\noperand tuples per primitive and prime width:")
        for name, per in COUNTS.items():
            print(f"  {name:26s} " + " ".join(f"{w}b:{c}" for w, c in sorted(per.items())))
    for name in ("fp_mulmod", "fp_mulmod_x", "fp_mulmod_term(even)", "fp_mulmod_term(odd)", "fp_mulmod2", "fp_renorm",
                 "fp_renorm_x", "fp_to_canonical<false>", "fp_to_canonical<true>", "shoup_mul_lazy", "shoup_mul",
                 "barrett64", "barrett128", "add_mod", "sub_mod", "neg_mod"):
        if name in COUNTS:
            low = {w: c for w, c in COUNTS[name].items() if c < N_PER_WIDTH}
            assert not low, (name, low)
