"""The bucket method (Pippenger, ecg_msm.cuh) at every window width, piece boundary and skew threshold on all twelve curves.

ecg_lincomb on n >= 2^13 terms cuts every scalar (secp256k1: every GLV half) into W windows of c bits, c = min(16,
max(8, floor(log2 nsub) - 5)) (P-521: c >= 9, msm_final_kernel runs one thread per window).  The width fixes the bucket
count, the top window's width (up to c + 1 bits, digits up to 2^(c+1)), the levels of the chunked running-sum reduction
and the Horner step.  Shards are cut into pieces of ECG_MSM_MAX_TERMS, and an input whose largest bucket holds more than
max(4096, 32 avg) points is declined and rerun per term.  So, on the device:

 A. every width c on every curve, n at an odd offset inside that width's range, each input mixing random scalars, k = 0,
    k = n - 1, identities at the head, tail and in a run, k P + (n - k) P pairs, P / -P pairs under equal scalars, and
    scalars that set every window below the top to 0, 1, 2^(c-1) - 1, 2^(c-1), 2^(c-1) + 1 and 2^c - 1 with and without
    an incoming carry, and the top window to its largest digit with and without one (secp256k1: on the GLV halves);
    lincomb_partial + point_sum at one width, lincomb through device pointers at the largest n;
 C. pieces of 2^13 terms whose last piece holds 1 to 33 terms (secp256k1's only route to c = 8), and the per-term path
    over two pieces of 2^20 terms;
 D. one bucket holding exactly the skew limit (bucket path) and one point more (declined, per-term path), for the
    absolute limit (P-256, c = 9) and the relative one (secp256k1 at 2^21 terms, c = 16).

The reference is exact at any n: every term takes a point of a pool P_j = [r_j] G with known r_j, so the sum is
[sum_i k_i r_j(i) mod n] G, one fixed-base multiplication (the scalar sums run on 16-bit limbs with np.bincount); once
per curve the terms condensed per pool point also go through ecref.lincomb.  Kernel-launch counts show which path ran.

Without a GPU: the geometry and recoder mirrors against tests/sim, the digit classes every case set reaches, the bucket
counts of the skew inputs, and the host twin of msm_run (tests/sim) at every forced width on every curve."""
import ctypes
import os
import random

import numpy as np
import pytest

import ecref
import pyref
from test_curves_ext import recs
from test_sim import sim  # noqa: F401  (fixture: builds tests/sim/libecgsim.so when stale)

NAMES = ["k256", "p256", "p384", "sm2", "bp256r1", "bp256t1", "bignp256", "bp384r1", "bp384t1", "p224", "p192", "p521"]
NL = {"k256": 8, "p256": 8, "p384": 12, "sm2": 8, "bp256r1": 8, "bp256t1": 8, "bignp256": 8, "bp384r1": 12, "bp384t1": 12,
      "p224": 7, "p192": 6, "p521": 17}
NT = os.cpu_count() or 4
POOL = 4096
MSM_MIN_TERMS = 1 << 13
MSM_MAX_TERMS = 1 << 24
FINAL_THREADS = 64
CH0, CHU = 16, 4
SKEW_ABS = 4096
LAMBDA = pyref.K256_LAMBDA


def _curve(name):
    return pyref.CURVES[name]


# ---------------------------------------------------------------------------------------------------------------------
# mirrors of msm_geometry / msm_run / lincomb_shard (ecgpu.cu) and msm_recode (ecg_msm.cuh)

def nbits(name):
    return 128 if name == "k256" else 32 * NL[name]


def geometry(name, n, c=None):
    """(c, W, nbits, nbw) as msm_geometry picks them for a piece of n terms (or at a given width c)"""
    nb = nbits(name)
    if c is None:
        nsub = 2 * n if name == "k256" else n
        c = min(16, max(8, nsub.bit_length() - 1 - 5))
        while -(-nb // c) > FINAL_THREADS:
            c += 1
    return c, -(-nb // c), nb, (1 << (c + 1)) + 2


def levels(c):
    """levels of the chunked running-sum reduction over the 2^(c+1) + 1 slots of a window"""
    ln, chl, lv = (1 << (c + 1)) + 1, CH0, 0
    while True:
        nch = -(-ln // chl)
        lv += 1
        if nch == 1:
            return lv
        ln, chl = nch, CHU


def bucket_launches(name, n, max_terms=MSM_MAX_TERMS):
    """kernels msm_run launches over the pieces of one shard (prep, three scan kernels, scatter, three order kernels,
    buckets, one per reduction level, final) plus the tree sum of the piece results"""
    cnts = [min(max_terms, n - lo) for lo in range(0, n, max_terms)]
    total = sum(10 + levels(geometry(name, cnt)[0]) for cnt in cnts)
    m = len(cnts)
    while m > 1:
        total += 1
        m = -(-m // 32)
    return total


def skew_limit(name, n):
    c = geometry(name, n)[0]
    nsub = 2 * n if name == "k256" else n
    return max(SKEW_ABS, 32 * (nsub // (1 << (c - 1)) + 1))


def widths(name):
    return list(range(9 if name in ("k256", "p521") else 8, 17))


def n_for(name, c):
    """n inside width c's range at an odd offset from a power of two: [2^(c+5), 2^(c+6)), secp256k1 [2^(c+4), 2^(c+5))"""
    return (1 << (c + (4 if name == "k256" else 5))) + 2 * c + 1


def recode(M16, c, nb):
    """msm_recode over the rows of M16 ((m, L) uint16 little-endian limbs of the magnitudes) -> (digits, raw window
    bits, incoming carry), each (m, W)"""
    W = -(-nb // c)
    h = 1 << (c - 1)
    m = M16.shape[0]
    M = np.zeros((m, max(M16.shape[1], (nb + 18) // 16) + 3), np.uint64)
    M[:, :M16.shape[1]] = M16

    def bits(pos, width):
        q, o = pos >> 4, pos & 15
        v = M[:, q] | (M[:, q + 1] << np.uint64(16)) | (M[:, q + 2] << np.uint64(32))
        return ((v >> np.uint64(o)) & np.uint64((1 << width) - 1)).astype(np.int64)

    D, R, CI = (np.zeros((m, W), np.int64) for _ in range(3))
    carry = np.zeros(m, np.int64)
    for w in range(W - 1):
        R[:, w] = bits(c * w, c)
        CI[:, w] = carry
        v = R[:, w] + carry
        big = v > h
        D[:, w] = np.where(big, v - (1 << c), v)
        carry = big.astype(np.int64)
    top = c * (W - 1)
    R[:, W - 1] = bits(top, min(17, nb + 1 - top))
    CI[:, W - 1] = carry
    D[:, W - 1] = R[:, W - 1] + carry
    return D, R, CI


def bucket_counts(D, nbw, weights=None):
    """points per (window, |digit|) bucket -> flat array over W * nbw slots"""
    m, W = D.shape
    a = np.abs(D)
    key = (np.arange(W)[None, :] * nbw + a).reshape(-1)
    wt = None if weights is None else np.repeat(np.asarray(weights, np.float64), W)
    cnt = np.bincount(key, weights=wt, minlength=W * nbw)
    cnt[np.arange(W) * nbw] = 0       # digit 0: no bucket
    return cnt.astype(np.int64)


# ---------------------------------------------------------------------------------------------------------------------
# limbs, records and the exact reference

def nlimbs(name):
    return pyref.fbytes(_curve(name)) // 2


def ints_to_limbs(vs, L):
    return np.frombuffer(b"".join(int(v).to_bytes(2 * L, "little") for v in vs), "<u2").reshape(-1, L).astype(np.uint16)


def records(name, K16):
    """(m, L) limbs -> (m, fbytes) scalar records in the curve's byte order"""
    b = np.ascontiguousarray(K16.astype("<u2")).view(np.uint8).reshape(K16.shape[0], -1)
    return b.copy() if _curve(name).le else np.ascontiguousarray(b[:, ::-1])


def random_limbs(rng, m, name, bits=None):
    """m random scalars below 2^bits (default bitlen(n) - 1, so below n)"""
    L, top = nlimbs(name), bits or _curve(name).n.bit_length() - 1
    K = rng.integers(0, 1 << 16, size=(m, L), dtype=np.uint32).astype(np.uint16)
    K[:, top // 16] &= np.uint16((1 << (top % 16)) - 1)
    K[:, top // 16 + 1:] = 0
    return K


_GLV_FILL = {}


def filler_limbs(rng, m, name, c):
    """m random scalars that leave every window not wholly below bit bitlen(n) - 1 (secp256k1: the top window of both
    GLV halves) at digit 0.  Such a window holds only the few top bits of n, at some widths 1 to 4 of them (P-521: the
    window across bit 521), so uniform scalars crowd its few buckets past the skew limit and the whole call is declined
    (P-256 at 2^16 terms: about 8200 points per top bucket); here only the case scalars reach those windows.
    secp256k1: a tile of 2^14 scalars built from random halves below 2^(top - 1), repeated."""
    _, W, _, _ = geometry(name, 0, c)
    top = c * (W - 1)
    if name != "k256":
        return random_limbs(rng, m, name, min(top, c * ((_curve(name).n.bit_length() - 1) // c)) - 1)
    if c not in _GLV_FILL:
        prng = random.Random(700 + c)
        n = pyref.K256.n
        ks = []
        while len(ks) < 1 << 14:
            k1, k2 = prng.getrandbits(top - 1) * prng.choice((1, -1)), prng.getrandbits(top - 1) * prng.choice((1, -1))
            k = (k1 + LAMBDA * k2) % n
            if pyref.glv_split(k) == (k1, k2):
                ks.append(k)
        _GLV_FILL[c] = ints_to_limbs(ks, 16)
    tile = _GLV_FILL[c]
    return tile[rng.permutation(np.arange(m) % tile.shape[0])]


_POOLS = {}


def pool(name):
    """4096 points P_j = [r_j] G per curve and session: (r, xy records, xy records of -P_j)"""
    if name not in _POOLS:
        c = _curve(name)
        rng = random.Random(4096 + NAMES.index(name))
        r = [rng.randrange(1, c.n) for _ in range(POOL)]
        xy, inf = ecref.mul_gen_batch(name, recs(c, r), nthreads=NT)
        assert not inf.any()
        nb = pyref.fbytes(c)
        xy = np.asarray(xy, np.uint8).reshape(POOL, 2 * nb)
        neg = xy.copy()
        for j in range(POOL):
            neg[j, nb:] = np.frombuffer(pyref.enc_fe(c, (c.p - pyref.dec_fe(c, xy[j, nb:].tobytes())) % c.p), np.uint8)
        _POOLS[name] = (r, xy, neg)
    return _POOLS[name]


class Terms:
    """n terms: scalar limbs K16, pool index, the point negated, the point the identity"""

    def __init__(self, K16, idx, neg, inf):
        self.K16, self.idx, self.neg, self.inf = K16, idx, neg, inf

    @property
    def n(self):
        return self.K16.shape[0]

    def arrays(self, name):
        """(scalar records, point records, identity flags) as ecg_lincomb takes them"""
        _, xy, nxy = pool(name)
        P = xy[self.idx]
        P[self.neg] = nxy[self.idx[self.neg]]
        P[self.inf] = 0
        return records(name, self.K16), P, self.inf.astype(np.uint8)

    def coefficients(self, name):
        """per pool point, the sum of its terms' scalars (negated for -P_j) mod n, by 16-bit limb sums"""
        c = _curve(name)
        bins = self.idx + POOL * self.neg.astype(np.int64)
        bins[self.inf] = 2 * POOL
        sums = [np.bincount(bins, weights=self.K16[:, q].astype(np.float64), minlength=2 * POOL + 1).astype(np.int64).tolist()
                for q in range(self.K16.shape[1])]   # at most 2^22 terms x 2^16: exact in float64
        S = [sum(sums[q][j] << (16 * q) for q in range(len(sums))) for j in range(2 * POOL)]
        return [(S[j] - S[POOL + j]) % c.n for j in range(POOL)]

    def expected(self, name):
        """[sum_i k_i r_j(i)] G as (xy record, identity flag), and that scalar"""
        c = _curve(name)
        r = pool(name)[0]
        t = sum(a * b for a, b in zip(self.coefficients(name), r)) % c.n
        xy, inf = ecref.mul_gen_batch(name, recs(c, [t]), nthreads=1)
        return (np.asarray(xy, np.uint8).reshape(-1), int(inf[0])), t


# ---------------------------------------------------------------------------------------------------------------------
# digit-boundary scalars

def window_values(c):
    h = 1 << (c - 1)
    return (0, 1, h - 1, h, h + 1, (1 << c) - 1)


def _set_window(k, w, c, v):
    return (k & ~(((1 << c) - 1) << (c * w))) | (v << (c * w))


def free_windows(name, c):
    """windows below the top whose every bit pattern is reachable: below bit bitlen(n) - 1 (GLV halves: below 2^125)"""
    _, W, _, _ = geometry(name, 0, c)
    bound = 125 if name == "k256" else _curve(name).n.bit_length() - 1
    return [w for w in range(W - 1) if c * (w + 1) <= bound]


def top_cases(name, c):
    """(T, carry-in reachable) of the top window, and the scalars that give it its largest digit with and without an
    incoming carry: T = the top bits of n - 1; a carry comes in exactly when the bits below exceed
    H = sum_w 2^(c-1) 2^(c w) (the largest value the signed windows hold without one)"""
    n = _curve(name).n
    _, W, _, _ = geometry(name, 0, c)
    top = c * (W - 1)
    T, L0 = (n - 1) >> top, (n - 1) & ((1 << top) - 1)
    H = (1 << (c - 1)) * ((1 << top) - 1) // ((1 << c) - 1)
    ks = [(T << top) | min(L0, H), (T << top) | (min(L0, H) >> 1)]
    if L0 > H:
        ks += [(T << top) | L0, (T << top) | (H + 1)]
    return T, L0 > H, ks


def boundary_scalars(name, c, seed=0):
    """non-GLV curves: every free window through window_values(c), the window below once giving a carry (2^(c-1) + 1) and
    once not (1), random bits elsewhere below bitlen(n) - 1; the top-window cases; n - 1 - i"""
    n = _curve(name).n
    bl = n.bit_length()
    rng = random.Random(seed * 100 + c * 7 + bl)
    out = []
    for w in free_windows(name, c):
        for v in window_values(c):
            for carry in ((0, 1) if w else (0,)):
                k = _set_window(rng.getrandbits(bl - 1), w, c, v)
                if w:
                    k = _set_window(k, w - 1, c, (1 << (c - 1)) + 1 if carry else 1)
                out.append(k)
    out += top_cases(name, c)[2]
    out += [n - 1 - i for i in range(16)] + [n - (1 << e) for e in range(0, bl - 1, 7)]
    return out


def _glv_try(rng, m, which, n):
    """a scalar whose model split has magnitude m in half `which` and a random other half (None if it does not)"""
    other = rng.getrandbits(124)
    s1, s2 = rng.choice((1, -1)), rng.choice((1, -1))
    k1, k2 = (s1 * m, s2 * other) if which == 0 else (s1 * other, s2 * m)
    k = (k1 + LAMBDA * k2) % n
    return k if pyref.glv_split(k) == (k1, k2) else None


_GLV_TOPS = {}


def _glv_top_scalars(c, count=6000):
    """random scalars whose halves give the top window its largest digits with and without an incoming carry"""
    if c not in _GLV_TOPS:
        n = pyref.K256.n
        rng = random.Random(9000 + c)
        ks = [rng.randrange(n) for _ in range(count)] + [n - 1 - i for i in range(64)]
        halves = [abs(h) for k in ks for h in pyref.glv_split(k)]
        D, _, CI = recode(ints_to_limbs(halves, 9), c, 128)
        best = {}
        for i in range(len(halves)):
            key = int(CI[i, -1])
            if key not in best or D[i, -1] > D[best[key], -1]:
                best[key] = i
        _GLV_TOPS[c] = [ks[i // 2] for i in best.values()]
    return _GLV_TOPS[c]


def glv_boundary_scalars(c, seed=0):
    """secp256k1: the patterns of boundary_scalars on each GLV half (kept where pyref.glv_split returns the intended
    halves), the top-window cases from the halves of random scalars, n - 1 - i"""
    n = pyref.K256.n
    rng = random.Random(seed * 100 + c)
    out = []
    for which in (0, 1):
        for w in free_windows("k256", c):
            for v in window_values(c):
                for carry in ((0, 1) if w else (0,)):
                    for _ in range(64):
                        m = _set_window(rng.getrandbits(124), w, c, v)
                        if w:
                            m = _set_window(m, w - 1, c, (1 << (c - 1)) + 1 if carry else 1)
                        k = _glv_try(rng, m, which, n)
                        if k is not None:
                            out.append(k)
                            break
                    else:
                        raise AssertionError(f"no scalar with half {which} window {w} = {v:#x}")
    return out + _glv_top_scalars(c) + [n - 1 - i for i in range(16)]


def case_scalars(name, c):
    return glv_boundary_scalars(c) if name == "k256" else boundary_scalars(name, c)


def magnitudes(name, ks):
    """what the prep kernel recodes: the scalars, or (secp256k1) the magnitudes of both GLV halves"""
    if name == "k256":
        return ints_to_limbs([abs(h) for k in ks for h in pyref.glv_split(k)], 9)
    return ints_to_limbs(ks, NL[name] * 2 + 2)


def build_terms(name, c, n, seed=1, pairs=256):
    """n terms at width c: the case scalars, k = 0 / n - 1, k P + (n - k) P pairs, P / -P pairs under equal scalars,
    identities at the head, the tail and in a run, random scalars on random pool points elsewhere"""
    cv = _curve(name)
    L = nlimbs(name)
    rng = np.random.default_rng(seed * 1000 + c)
    prng = random.Random(seed * 1000 + c)
    K = filler_limbs(rng, n, name, c)
    idx = rng.integers(0, POOL, n)
    neg = np.zeros(n, bool)
    inf = np.zeros(n, bool)
    spec = case_scalars(name, c) + [0, 0, cv.n - 1, 1]
    pos = 8
    K[pos:pos + len(spec)] = ints_to_limbs(spec, L)
    pos += len(spec)
    ks = [prng.randrange(1, cv.n) for _ in range(pairs)]            # k P + (n - k) P
    K[pos:pos + 2 * pairs:2] = ints_to_limbs(ks, L)
    K[pos + 1:pos + 2 * pairs:2] = ints_to_limbs([cv.n - k for k in ks], L)
    idx[pos + 1:pos + 2 * pairs:2] = idx[pos:pos + 2 * pairs:2]
    pos += 2 * pairs
    K[pos + 1:pos + 2 * pairs:2] = K[pos:pos + 2 * pairs:2]         # P and -P, equal scalars
    idx[pos + 1:pos + 2 * pairs:2] = idx[pos:pos + 2 * pairs:2]
    neg[pos + 1:pos + 2 * pairs:2] = True
    pos += 2 * pairs
    assert pos + 100 < n - 3
    inf[:3] = True
    inf[-3:] = True
    inf[pos:pos + 100] = True
    return Terms(K, idx, neg, inf)


def _same(got, want):
    return np.array_equal(np.asarray(got[0], np.uint8).reshape(-1), want[0]) and int(got[1]) == want[1]


# ---------------------------------------------------------------------------------------------------------------------
# skew inputs

SKEW_DIGIT = 0xB3


def skew_terms_p256(extra):
    """P-256 at n = 2^14 (c = 9, the absolute limit 4096 binds): 4096 + extra terms with window-0 bits SKEW_DIGIT (digit
    +SKEW_DIGIT), the rest avoiding SKEW_DIGIT and 2^9 - SKEW_DIGIT (digit -SKEW_DIGIT) there"""
    name, n = "p256", 1 << 14
    rng = np.random.default_rng(77)
    K = random_limbs(rng, n, name)
    low = K[:, 0].astype(np.int64)
    w0 = low & 0x1FF
    bad = (w0 == SKEW_DIGIT) | (w0 == 512 - SKEW_DIGIT)
    K[bad, 0] ^= np.uint16(1 << 4)
    m = SKEW_ABS + extra
    K[:m, 0] = (K[:m, 0] & np.uint16(0xFE00)) | np.uint16(SKEW_DIGIT)
    return Terms(K, rng.integers(0, POOL, n), np.zeros(n, bool), np.zeros(n, bool))


SKEW_LOW16 = 0x2B6D
_K256_TILE = {}


def _k256_tile(size=1 << 14):
    """random secp256k1 scalars none of whose GLV halves has window-0 digit +-SKEW_LOW16 at c = 16, and their halves"""
    if size not in _K256_TILE:
        n = pyref.K256.n
        rng = random.Random(2121)
        ks = [rng.randrange(n) for _ in range(size + 64)]
        halves = [abs(h) for k in ks for h in pyref.glv_split(k)]
        D = recode(ints_to_limbs(halves, 9), 16, 128)[0]
        ok = ~(np.abs(D[:, 0]) == SKEW_LOW16).reshape(-1, 2).any(axis=1)
        ks = [k for k, g in zip(ks, ok) if g][:size]
        _K256_TILE[size] = (ks, ints_to_limbs([abs(h) for k in ks for h in pyref.glv_split(k)], 9))
    return _K256_TILE[size]


def skew_terms_k256(extra):
    """secp256k1 at n = 2^21 (c = 16, relative limit 32 (2^22 / 2^15 + 1) = 4128): 4128 + extra scalars below 2^120
    (k2 = 0, so their window-0 digit is their low 16 bits) with low bits SKEW_LOW16, the rest a tile of 2^14 random
    scalars repeated"""
    name, n = "k256", 1 << 21
    m = skew_limit(name, n) + extra
    tile, _ = _k256_tile()
    rng = np.random.default_rng(2122)
    prng = random.Random(2123)
    small = [(prng.getrandbits(104) << 16) | SKEW_LOW16 for _ in range(m)]
    reps = -(-(n - m) // len(tile))
    tl = np.tile(ints_to_limbs(tile, 16), (reps, 1))[:n - m]
    K = np.concatenate([ints_to_limbs(small, 16), tl])
    return Terms(K, rng.integers(0, POOL, n), np.zeros(n, bool), np.zeros(n, bool)), small


def skew_counts(name, T, small=None):
    """largest bucket and the bucket count at the skew digit, from the recoder mirror"""
    if name == "p256":
        c, W, nb, nbw = geometry(name, T.n)
        D = recode(T.K16, c, nb)[0]
        cnt = bucket_counts(D[~T.inf], nbw)
        return int(cnt.max()), int(cnt[SKEW_DIGIT])
    c, W, nb, nbw = geometry(name, T.n)
    tile, halves = _k256_tile()
    m = len(small)
    reps = np.bincount(np.arange(T.n - m) % len(tile), minlength=len(tile))
    Dt = recode(halves, c, nb)[0]
    cnt = bucket_counts(Dt, nbw, np.repeat(reps, 2))
    Ds = recode(ints_to_limbs(small, 9), c, nb)[0]               # k1 = k, k2 = 0 (no digits)
    cnt += bucket_counts(Ds, nbw)
    return int(cnt.max()), int(cnt[SKEW_LOW16])


# ---------------------------------------------------------------------------------------------------------------------
# A. every width on every curve (GPU)

@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_every_width(engine, name):
    """lincomb at every reachable c against [sum k_i r_j(i)] G; the launch count of the bucket path alone; at the
    largest width also ecref.lincomb over the terms condensed per pool point and (secp256k1, P-384, P-521) the same call
    through device pointers; lincomb_partial of two halves + point_sum at the second width"""
    ws = widths(name)
    tail = None
    for c in ws:
        n = n_for(name, c)
        assert geometry(name, n)[0] == c
        T = build_terms(name, c, n)
        K, P, I = T.arrays(name)
        want, t = T.expected(name)
        l0 = engine.kernel_launches
        got = engine.lincomb(name, K, P, I)
        launches = engine.kernel_launches - l0
        if tail is None:
            tail = launches - bucket_launches(name, n)       # the normalisation of the result
            assert 1 <= tail <= 2, f"{name}: {launches} launches at n = {n}"
        assert launches == bucket_launches(name, n) + tail, f"{name} c = {c}: not the bucket path alone ({launches} launches)"
        assert _same(got, want), f"{name} c = {c} n = {n}: lincomb != [{t:#x}] G"
        if c == ws[1]:
            h = n // 2
            fb = pyref.fbytes(_curve(name))
            p1 = engine.lincomb_partial(name, K[:h], P[:h], I[:h])
            p2 = engine.lincomb_partial(name, K[h:], P[h:], I[h:])
            assert _same(engine.point_sum(name, np.concatenate([p1, p2])), want), f"{name} c = {c}: lincomb_partial + point_sum"
            assert p1.size == 3 * fb
        if c == ws[-1]:
            cv = _curve(name)
            ref = ecref.lincomb(name, recs(cv, T.coefficients(name)), pool(name)[1].reshape(-1), np.zeros(POOL, np.uint8), nthreads=NT)
            assert _same(ref, want), f"{name}: the condensed ecref.lincomb disagrees with the fixed-base reference"
            if name in ("k256", "p384", "p521"):
                _lincomb_device_pointers(name, K, P, I, want)
        del K, P, I, T


def _lincomb_device_pointers(name, K, P, I, want):
    import torch

    import ecgpu

    fb = pyref.fbytes(_curve(name))
    dev = torch.device("cuda:0")
    eng = ecgpu.Engine([0], device_ptrs=True)
    try:
        kd, pd, idd = (torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).to(dev) for a in (K, P, I))
        oxy = torch.full((2 * fb,), 0xAA, dtype=torch.uint8, device=dev)
        oinf = torch.full((1,), 0xAA, dtype=torch.uint8, device=dev)
        eng.lincomb_ptr(name, K.shape[0], kd.data_ptr(), pd.data_ptr(), idd.data_ptr(), oxy.data_ptr(), oinf.data_ptr())
        torch.cuda.synchronize()
        assert _same((oxy.cpu().numpy(), int(oinf.cpu()[0])), want), f"{name}: lincomb through device pointers"
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# C. piece boundaries (GPU)

PIECE = 1 << 13
PIECE_NS = [PIECE + r for r in (1, 2, 31, 32, 33)] + [3 * PIECE + 1]


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_piece_boundaries(engine, monkeypatch, name):
    """pieces of 2^13 terms whose last piece holds 1, 2, 31, 32 or 33 terms (and 3 full pieces + 1): every piece through
    the bucket method, the piece sums added by the tree sum"""
    monkeypatch.setenv("ECG_MSM_MAX_TERMS", str(PIECE))
    c0 = widths(name)[0]
    tail = None
    for n in PIECE_NS:
        T = build_terms(name, c0, n, seed=3, pairs=64)
        K, P, I = T.arrays(name)
        want, t = T.expected(name)
        l0 = engine.kernel_launches
        got = engine.lincomb(name, K, P, I)
        launches = engine.kernel_launches - l0
        expect = bucket_launches(name, n, PIECE)
        if tail is None:
            tail = launches - expect
            assert 1 <= tail <= 2, f"{name}: {launches} launches at n = {n}"
        assert launches == expect + tail, f"{name} n = {n}: {launches} launches, the pieces' bucket paths take {expect + tail}"
        assert _same(got, want), f"{name} n = {n} in pieces of {PIECE}: lincomb != [{t:#x}] G"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["k256", "p256", "p384", "bp256r1"])
def test_per_term_two_pieces(name):
    """the constant-time context forces the per-term path: n = 2^20 + 3 runs two pieces, the second of three terms"""
    import ecgpu

    n = (1 << 20) + 3
    T = build_terms(name, widths(name)[-1], n, seed=5)
    T.K16[-3:] = ints_to_limbs([0, _curve(name).n - 1, 12345], nlimbs(name))
    T.inf[-3:] = False
    K, P, I = T.arrays(name)
    want, t = T.expected(name)
    eng = ecgpu.Engine(consttime=True)
    try:
        got = eng.lincomb(name, K, P, I)
    finally:
        eng.close()
    assert _same(got, want), f"{name}: per-term lincomb over two pieces != [{t:#x}] G"


# ---------------------------------------------------------------------------------------------------------------------
# D. skew thresholds at their boundary (GPU)

def _skew_run(engine, name, inputs, limit):
    """inputs: [(terms, largest bucket)]; the first at the limit must stay on the bucket path, the second be declined"""
    base = None
    for T, biggest in inputs:
        K, P, I = T.arrays(name)
        want, t = T.expected(name)
        if base is None:   # a random input of the same size: the launch count of the bucket path alone
            R = Terms(random_limbs(np.random.default_rng(5), T.n, name), T.idx, T.neg, T.inf)
            l0 = engine.kernel_launches
            engine.lincomb(name, records(name, R.K16), P, I)
            base = engine.kernel_launches - l0
        l0 = engine.kernel_launches
        got = engine.lincomb(name, K, P, I)
        launches = engine.kernel_launches - l0
        assert _same(got, want), f"{name}: largest bucket {biggest}: lincomb != [{t:#x}] G"
        if biggest <= limit:
            assert launches == base, f"{name}: a bucket of {biggest} <= {limit} points was declined ({launches} launches, bucket path {base})"
        else:
            assert launches > base, f"{name}: a bucket of {biggest} > {limit} points stayed on the bucket path"


@pytest.mark.gpu
def test_skew_absolute_limit(engine):
    limit = skew_limit("p256", 1 << 14)
    assert limit == SKEW_ABS
    inputs = []
    for extra in (0, 1):
        T = skew_terms_p256(extra)
        biggest, at = skew_counts("p256", T)
        assert biggest == at == SKEW_ABS + extra
        inputs.append((T, biggest))
    _skew_run(engine, "p256", inputs, limit)


@pytest.mark.gpu
def test_skew_relative_limit(engine):
    limit = skew_limit("k256", 1 << 21)
    assert limit == 4128
    inputs = []
    for extra in (0, 1):
        T, small = skew_terms_k256(extra)
        biggest, at = skew_counts("k256", T, small)
        assert biggest == at == limit + extra
        inputs.append((T, biggest))
    _skew_run(engine, "k256", inputs, limit)


# ---------------------------------------------------------------------------------------------------------------------
# without a GPU: mirrors against the host simulation, case coverage, skew counts, the host twin at every width

def _sim_geometry(sim, name, n):
    out = (ctypes.c_int * 4)()
    sim.sim_msm_geometry(pyref.CURVE_IDS[name], ctypes.c_size_t(n), out)
    return tuple(out)


@pytest.mark.parametrize("name", NAMES)
def test_geometry_mirror_matches_sim(sim, name):
    ns = sorted({max(1, (1 << e) + d) for e in range(0, 26) for d in (-1, 0, 1, 3)})
    for n in ns:
        assert geometry(name, n) == _sim_geometry(sim, name, n), (name, n)
    for c in widths(name):
        n = n_for(name, c)
        assert n % 2 == 1 and geometry(name, n)[0] == c and n >= MSM_MIN_TERMS
        e = c + (4 if name == "k256" else 5)
        assert 1 << e <= n < 1 << (e + 1)
    assert geometry(name, (1 << 21) + 1)[0] == 16
    if name == "k256":   # c = 8 only through a piece tail
        assert geometry(name, MSM_MIN_TERMS)[0] == 9 and geometry(name, 33)[0] == 8
    if name == "p521":
        assert geometry(name, MSM_MIN_TERMS)[0] == 9 and geometry(name, 1)[0] == 9


@pytest.mark.parametrize("name", NAMES)
def test_recode_mirror_matches_sim(sim, name):
    """the recoder mirror against msm_recode on the case scalars (secp256k1: their halves) and random magnitudes"""
    nb = nbits(name)
    nm = 9 if name == "k256" else NL[name] + 1
    rng = np.random.default_rng(3)
    for c in ([8] if name == "k256" else []) + widths(name):
        M = magnitudes(name, case_scalars(name, c)[::5])
        R = rng.integers(0, 1 << 16, size=(200, M.shape[1]), dtype=np.uint32).astype(np.uint16)
        R[:, (nb + 1) // 16:] = 0
        M = np.concatenate([M, R])
        D = recode(M, c, nb)[0]
        Mp = np.zeros((M.shape[0], 2 * nm), "<u2")
        Mp[:, :min(2 * nm, M.shape[1])] = M[:, :2 * nm]
        M32 = Mp.view("<u4")
        out = np.zeros(D.shape[1], np.int32)
        for i in range(M.shape[0]):
            row = np.ascontiguousarray(M32[i])
            W = sim.sim_msm_recode_n(row.ctypes.data_as(ctypes.c_void_p), nm, c, nb, out.ctypes.data_as(ctypes.c_void_p))
            assert W == D.shape[1]
            assert np.array_equal(out, D[i]), (name, c, i)


def _coverage(name, c):
    nb = nbits(name)
    D, R, CI = recode(magnitudes(name, case_scalars(name, c)), c, nb)
    return D, R, CI


@pytest.mark.parametrize("name", NAMES)
def test_case_sets_reach_every_digit_class(sim, name):
    """for every width: every free window below the top holds each boundary value with and without an incoming carry;
    the top window reaches its largest digit with and without a carry (above 2^(c-1) where the curve allows it); the
    secp256k1 halves are the ones the device split produces"""
    above = []
    for c in widths(name):
        D, R, CI = _coverage(name, c)
        W = D.shape[1]
        seen = set(zip(np.nonzero(np.ones_like(R, bool))[1].tolist(), R.reshape(-1).tolist(), CI.reshape(-1).tolist()))
        for w in free_windows(name, c):
            for v in window_values(c):
                for carry in ((0, 1) if w else (0,)):
                    assert (w, v, carry) in seen, f"{name} c = {c}: window {w} value {v:#x} carry {carry} not reached"
        topd, topc = D[:, -1], CI[:, -1]
        if name == "k256":
            assert (topc == 1).any() and (topc == 0).any()
            best = int(topd.max())
        else:
            T, carry_in, _ = top_cases(name, c)
            best = T + int(carry_in)
            assert int(topd.max()) == best, f"{name} c = {c}: largest top digit {int(topd.max())}, reachable {best}"
            assert (topd[topc == 0] == T).any()
            if carry_in:
                assert (topd[topc == 1] == T + 1).any()
        if best > 1 << (c - 1):
            above.append(c)
    # the top window's buckets above 2^(c-1) (the slots msm_wreduce_kernel reads only in the top row)
    want = {"k256": {16}, "p521": set(), "p384": {8, 12, 16}, "bp384r1": {8, 12, 16}, "bp384t1": {8, 12, 16},
            "p224": {8, 14, 16}, "p192": {8, 12, 16}}.get(name, {8, 16})
    assert want <= set(above), f"{name}: top digits above 2^(c-1) at c = {above}"
    if name == "k256":   # the halves of the case scalars are the device's: glv_split_k256 on the host
        ks = case_scalars(name, 12)[::7]
        out = np.zeros(36, np.uint8)
        for k in ks:
            sim.sim_k256_glv(np.frombuffer(k.to_bytes(32, "big"), np.uint8).ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p))
            h1 = 2 * int.from_bytes(out[:16].tobytes(), "little") + 1 - int(out[17])
            h2 = 2 * int.from_bytes(out[18:34].tobytes(), "little") + 1 - int(out[35])
            k1, k2 = pyref.glv_split(k)
            assert (h1, h2) == (abs(k1), abs(k2)) and (out[16], out[34]) == (k1 < 0, k2 < 0), hex(k)


def test_skew_inputs_hold_the_limit():
    """the bucket counts of section D's inputs: exactly the limit, and one more, in the bucket of the chosen digit"""
    for extra in (0, 1):
        T = skew_terms_p256(extra)
        assert skew_counts("p256", T) == (SKEW_ABS + extra, SKEW_ABS + extra)
    limit = skew_limit("k256", 1 << 21)
    assert limit == 32 * ((1 << 22) // (1 << 15) + 1) == 4128
    for extra in (0, 1):
        T, small = skew_terms_k256(extra)
        assert T.n == 1 << 21
        assert skew_counts("k256", T, small) == (limit + extra, limit + extra)
    # small scalars: k1 = k, k2 = 0 under the model split (k g / 2^384 rounds to 0 below 2^120)
    for k in small[:64] + [(1 << 120) - 1]:
        assert pyref.glv_split(k) == (k, 0)


def _sim_lincomb(sim, name, T, c):
    K, P, I = T.arrays(name)
    fb = pyref.fbytes(_curve(name))
    oxy, oinf, st, path = np.zeros(2 * fb, np.uint8), np.zeros(1, np.uint8), np.zeros(2, np.uint32), ctypes.c_int(-1)
    sim.simk_lincomb_c(pyref.CURVE_IDS[name], ctypes.c_size_t(T.n), _ptr(K), _ptr(P), _ptr(I), ctypes.c_size_t(64), _ptr(oxy), _ptr(oinf),
                       _ptr(st), ctypes.byref(path), 1, c)
    assert st[0] == 0
    return (oxy, int(oinf[0])), path.value


def _ptr(a):
    return np.ascontiguousarray(a).ctypes.data_as(ctypes.c_void_p)


def small_terms(name, c, n=300, seed=7):
    """a few hundred terms at width c: a sample of the case scalars, pairs, identities"""
    cv = _curve(name)
    rng = np.random.default_rng(seed + c)
    prng = random.Random(seed + c)
    L = nlimbs(name)
    spec = case_scalars(name, c)
    spec = prng.sample(spec, min(len(spec), n // 2)) + top_cases(name, c)[2] * (name != "k256") + [0, cv.n - 1]
    K = random_limbs(rng, n, name)
    K[3:3 + len(spec)] = ints_to_limbs(spec, L)
    idx = rng.integers(0, 64, n)
    neg = np.zeros(n, bool)
    inf = np.zeros(n, bool)
    p = 3 + len(spec)
    ks = [prng.randrange(1, cv.n) for _ in range(10)]
    K[p:p + 20:2], K[p + 1:p + 20:2] = ints_to_limbs(ks, L), ints_to_limbs([cv.n - k for k in ks], L)
    idx[p + 1:p + 20:2] = idx[p:p + 20:2]
    K[p + 21:p + 40:2] = K[p + 20:p + 40:2]
    idx[p + 21:p + 40:2] = idx[p + 20:p + 40:2]
    neg[p + 21:p + 40:2] = True
    inf[:2] = inf[-2:] = True
    inf[p + 40:p + 45] = True
    return Terms(K, idx, neg, inf)


@pytest.mark.parametrize("name", NAMES)
def test_host_twin_every_width(sim, name):
    """msm_run's kernel chain on the host (tests/sim simk_lincomb_c) with c forced to every width: scan, scatter,
    ordering, the recursive weighted reduction and Horner at each geometry"""
    # P-521 stops at c = 15: its 34 windows of 2^17 slots at c = 16 take about a minute in the simulation
    for c in (range(9, 16) if name == "p521" else range(8, 17)):
        T = small_terms(name, c)
        want, t = T.expected(name)
        got, path = _sim_lincomb(sim, name, T, c)
        assert path == 1, f"{name} c = {c}: path {path}"
        assert _same(got, want), f"{name} c = {c}: host twin != [{t:#x}] G"
    cv = _curve(name)   # the fixed-base reference against ecref.lincomb over the condensed terms
    ref = ecref.lincomb(name, recs(cv, T.coefficients(name)), pool(name)[1].reshape(-1), np.zeros(POOL, np.uint8), nthreads=NT)
    assert _same(ref, want)
