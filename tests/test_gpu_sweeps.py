"""Dense sweeps of every curve's device kernels through the scalars and batch layouts where their rare branches run.

Random scalars almost never reach the exceptional endings of the window loops (the accumulator meeting plus or minus the
table entry, the parity correction from the identity), and small batches never put more than one element in a thread's
slice of the strided Montgomery-trick kernels.  So, on the device, for all twelve curves:

 A. scalar sweeps: every k below 1024 and above n - 1024, 2^e - 1 / 2^e / 2^e + 1 / n - 2^e for every e below the bit
    length of n, every 4-bit window of the variable-base recoding and every 16-bit window of the fixed-base recoding
    through its boundary values, and (secp256k1) neighbours of multiples of lambda, where one GLV half is tiny or zero;
    through k*P (P = G, a random point, the identity), the x-only entry, the constant-time context, k*G, and a*G + b*P
    ending in the identity or in a doubling;
 B. identities and refused entries inside the slices of normalize_kernel, ecdsa_prep_kernel / ecdsa_prep_generic_kernel and
    ecdsa_recover_prep_kernel, at slice heads, tails, whole slices, runs, every third element and the whole batch, with
    slice sizes from 1 to 33 elements per inversion;
 C. the bucket method (2^14 + 3 terms) on cancelling pairs, repeated points (the doubling branch inside a bucket) and
    P / -P with equal digits (a bucket that reaches the identity partway through).

Every output is compared byte for byte with the C restatements (oracle/ecref*.c) or, where those have no entry, with sums
and verdicts of the big-integer model (oracle/pyref.py).  The case builders and verdict rules run without a GPU too."""
import math
import os
import random

import numpy as np
import pytest

import ecref
import pyref
from test_curves_ext import pts, recs

NAMES = ["k256", "p256", "p384", "sm2", "bp256r1", "bp256t1", "bignp256", "bp384r1", "bp384t1", "p224", "p192", "p521"]
ECDSA_NAMES = ["k256", "p256", "p192", "p224", "p384", "p521", "bp256r1", "bp256t1", "bp384r1", "bp384t1"]
NT = os.cpu_count() or 4
K256_LAMBDA = pyref.K256_LAMBDA


def _curve(name):
    return pyref.CURVES[name]


def _fb(c):
    return pyref.fbytes(c)


def _uniq(ks):
    return list(dict.fromkeys(ks))


def _below(n, k):
    """k kept below n: first drop the fill's top bit, then reduce (patterns in the top window may still exceed n)"""
    if k >= n:
        k &= ~(1 << (n.bit_length() - 1))
    return k % n


# ---------------------------------------------------------------------------------------------------------------------
# A. scalar sets

def scalar_set(name, seed=0):
    """the variable-base sweep set S of one curve (every element below n)"""
    c = _curve(name)
    n, bl = c.n, c.n.bit_length()
    rng = random.Random(seed * 1000 + bl)
    ks = list(range(1024)) + [n - i for i in range(1, 1024)]
    for e in range(bl):
        ks += [(1 << e) - 1, 1 << e, ((1 << e) + 1) % n, n - (1 << e)]
    full = (1 << bl) - 1
    for w in range((bl + 3) // 4):        # every 4-bit window of the signed radix-16 recoding
        for fill in (0, full, rng.getrandbits(bl)):
            for v in (0x0, 0x1, 0x7, 0x8, 0x9, 0xF):
                ks.append(_below(n, (fill & ~(0xF << (4 * w))) | (v << (4 * w))))
    if name == "k256":                    # one GLV half tiny or zero
        for m in range(1, 41):
            for d in (-2, -1, 0, 1, 2):
                ks += [(m * K256_LAMBDA + d) % n, (n - m * K256_LAMBDA + d) % n]
    return _uniq(ks)


FB_PATTERNS = (0x0000, 0x0001, 0x7FFF, 0x8000, 0x8001, 0xFFFE, 0xFFFF)


def fixedbase_windows(name):
    return (_curve(name).n.bit_length() + 15) // 16


def fixedbase_patterns(name, seed=0):
    """[(k, window, pattern, fill kind)]: every 16-bit window below the bit length of n (P-224: 14, P-521: 33 with a
    9-bit top window) through the boundary values of the signed odd 16-bit digits, with zero / all-ones / random fill"""
    c = _curve(name)
    n, bl = c.n, c.n.bit_length()
    rng = random.Random(seed * 7 + bl)
    out = []
    for w in range(fixedbase_windows(name)):
        width = min(16, bl - 16 * w)
        for v in FB_PATTERNS:
            v &= (1 << width) - 1
            for kind, fill in (("0", 0), ("1", (1 << bl) - 1), ("r", rng.getrandbits(bl))):
                out.append((_below(n, (fill & ~(0xFFFF << (16 * w))) | (v << (16 * w))), w, v, kind))
    return out


def _first_bad(got_xy, got_inf, want_xy, want_inf):
    m = got_inf.size
    g, w = np.asarray(got_xy).reshape(m, -1), np.asarray(want_xy).reshape(m, -1)
    return np.nonzero((g != w).any(axis=1) | (np.asarray(got_inf).reshape(-1) != np.asarray(want_inf).reshape(-1)))[0]


def _assert_same(what, ks, got, want):
    bad = _first_bad(got[0], got[1], want[0], want[1])
    assert not bad.size, f"{what}: {bad.size}/{len(ks)} wrong, first at k = {[hex(ks[i]) for i in bad[:6]]}"


def _sample(ks):
    """positions checked against the big-integer model as well"""
    m = len(ks)
    return sorted(set([0, 1, 2, 3, 1023, 1024, 1025, 2045, 2046] + [m - 1, m - 2, m // 2]))


@pytest.fixture(scope="module")
def ct_engine():
    import ecgpu

    eng = ecgpu.Engine(consttime=True)
    yield eng
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_varbase_scalar_sweep(engine, ct_engine, name):
    """k*P over S for P = G, a random point and the identity; the x-only entry and the constant-time context give the
    same bytes"""
    c = _curve(name)
    nb = _fb(c)
    ks = scalar_set(name)
    m = len(ks)
    K = recs(c, ks)
    rng = random.Random(77)
    P = pyref.mul(c, rng.randrange(1, c.n), pyref.G(c))
    for label, pt in (("G", pyref.G(c)), ("P", P), ("O", None)):
        pxy, pinf = pts(c, [pt] * m)
        got = engine.mul_batch(name, K, pxy, pinf)
        want = ecref.mul_batch(name, K, pxy, pinf, nthreads=NT)
        _assert_same(f"{name} k*{label}", ks, got, want)
        if pt is None:
            assert got[1].all() and not np.asarray(got[0]).any()
        else:
            assert [int(i) for i in np.nonzero(got[1])[0]] == [i for i, k in enumerate(ks) if k == 0]
            xy = np.asarray(got[0]).reshape(m, 2 * nb)
            for i in _sample(ks):
                w = pyref.mul(c, ks[i], pt)
                assert (None if got[1][i] else (pyref.dec_fe(c, xy[i, :nb].tobytes()), pyref.dec_fe(c, xy[i, nb:].tobytes()))) == w, i
        x, xinf = engine.mul_batch_x(name, K, pxy, pinf)
        assert np.array_equal(x, np.asarray(got[0]).reshape(m, 2 * nb)[:, :nb]) and np.array_equal(xinf, got[1]), f"{name} x-only k*{label}"
        _assert_same(f"{name} constant-time k*{label}", ks, ct_engine.mul_batch(name, K, pxy, pinf), want)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_fixedbase_window_sweep(engine, ct_engine, name):
    """k*G over S and over every 16-bit window pattern: the fixed-base kernel and the constant-time context (k*G through
    the variable-base routine) against the C restatement; the identity exactly where k = 0"""
    c = _curve(name)
    cases = fixedbase_patterns(name)
    ks = _uniq(scalar_set(name) + [k for k, *_ in cases])
    K = recs(c, ks)
    want = ecref.mul_gen_batch(name, K, nthreads=NT)
    got = engine.mul_by_generator(name, K)
    bad = _first_bad(got[0], got[1], want[0], want[1])
    if bad.size:
        where = {k: (w, v, f) for k, w, v, f in cases}
        detail = [(hex(ks[i]), where.get(ks[i])) for i in bad[:8]]
        pytest.fail(f"{name} k*G: {bad.size}/{len(ks)} wrong, first (k, (window, pattern, fill)) = {detail}")
    assert [int(i) for i in np.nonzero(got[1])[0]] == [i for i, k in enumerate(ks) if k == 0]
    _assert_same(f"{name} constant-time k*G", ks, ct_engine.mul_by_generator(name, K), want)


def mul_gen_add_cases(name, count=64, seed=5):
    """(a, b, P, expected kind): b = -a t^-1 with P = t G ends at the identity, b = a t^-1 at a doubling of a G"""
    c = _curve(name)
    n = c.n
    rng = random.Random(seed)
    ts = [rng.randrange(1, n) for _ in range(count)]
    txy, tinf = ecref.mul_gen_batch(name, recs(c, ts), nthreads=NT)
    nb = _fb(c)
    txy = np.asarray(txy).reshape(count, 2 * nb)
    out = []
    for i, t in enumerate(ts):
        P = (pyref.dec_fe(c, txy[i, :nb].tobytes()), pyref.dec_fe(c, txy[i, nb:].tobytes()))
        a = rng.randrange(1, n)
        ti = pow(t, -1, n)
        out.append((a, (-a * ti) % n, P, "identity"))
        out.append((a, a * ti % n, P, "double"))
    P0 = out[0][2]
    out += [(0, rng.randrange(1, n), P0, "b*P"), (rng.randrange(1, n), 0, P0, "a*G"), (rng.randrange(1, n), rng.randrange(1, n), None, "a*G"),
            (0, 0, P0, "identity"), (0, 0, None, "identity"), (n - 1, 1, pyref.G(c), "identity"), (1, 1, pyref.G(c), "double")]
    return out


def _model_sum(name, cases):
    """a*G + b*P as the model sum of two C outputs"""
    c = _curve(name)
    nb = _fb(c)
    A, B = recs(c, [x[0] for x in cases]), recs(c, [x[1] for x in cases])
    pxy, pinf = pts(c, [x[2] for x in cases])
    gxy, ginf = ecref.mul_gen_batch(name, A, nthreads=NT)
    qxy, qinf = ecref.mul_batch(name, B, pxy, pinf, nthreads=NT)
    gxy, qxy = np.asarray(gxy).reshape(-1, 2 * nb), np.asarray(qxy).reshape(-1, 2 * nb)

    def dec(xy, inf, i):
        return None if inf[i] else (pyref.dec_fe(c, xy[i, :nb].tobytes()), pyref.dec_fe(c, xy[i, nb:].tobytes()))

    return [pyref.add(c, dec(gxy, ginf, i), dec(qxy, qinf, i)) for i in range(len(cases))], (A, B, pxy, pinf)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_mul_gen_add_exceptional_endings(engine, name):
    c = _curve(name)
    nb = _fb(c)
    cases = mul_gen_add_cases(name)
    want, (A, B, pxy, pinf) = _model_sum(name, cases)
    xy, inf = engine.mul_by_generator_and_mul_add(name, A, B, pxy, pinf)
    xy = np.asarray(xy).reshape(-1, 2 * nb)
    got = [None if inf[i] else (pyref.dec_fe(c, xy[i, :nb].tobytes()), pyref.dec_fe(c, xy[i, nb:].tobytes())) for i in range(len(cases))]
    bad = [(i, cases[i][3]) for i in range(len(cases)) if got[i] != want[i]]
    assert not bad, f"{name} a*G + b*P: {len(bad)} wrong, first {bad[:6]}"
    assert all(w is None for (*_, kind), w in zip(cases, want) if kind == "identity")
    assert all(not xy[i].any() for i in range(len(cases)) if inf[i])


# ---------------------------------------------------------------------------------------------------------------------
# B. slice layouts of the strided Montgomery-trick kernels
#
# Mirrors of ecgpu.cu: the thread count of normalize_kernel (launch_normalize and ensure_fb_table:
#   want = max(ceil(n / 32), min(n, SMs * 256)), 256-thread blocks),
# of ecdsa_prep_kernel / ecdsa_prep_generic_kernel / ecdsa_recover_prep_kernel (run_chunk:
#   want = max(ceil(n / 32), min(n, SMs * 128)), 128-thread blocks),
# where T = the launched grid (want rounded up to whole blocks); and the host-mode chunk schedule (chunk_schedule, with
# wave = SMs x vb_minblk x vb_block of the curve).  Thread t of a launch over a chunk owns t, t + T, t + 2T, ...

HOST_CHUNK = 1 << 18
DEV_CHUNK = 1 << 22
_NL = {"k256": 8, "p256": 8, "p384": 12, "sm2": 8, "bp256r1": 8, "bp256t1": 8, "bignp256": 8, "bp384r1": 12, "bp384t1": 12,
       "p224": 7, "p192": 6, "p521": 17}


def per_sm(name):
    """resident blocks x block size of the curve's variable-base kernel (vb_minblk x vb_block)"""
    if name == "k256":
        return 2 * 256
    if name == "p256":
        return 5 * 128
    if name == "p384":
        return 3 * 128
    nl = _NL[name]
    return (2 if nl > 12 else 3 if nl > 8 else 4) * 128


def _threads(cnt, sms, block):
    want = max((cnt + 31) // 32, min(cnt, sms * block))
    return (want + block - 1) // block * block


def norm_threads(cnt, sms):
    return _threads(cnt, sms, 256)


def prep_threads(cnt, sms):
    return _threads(cnt, sms, 128)


def host_chunks(n, wave):
    """chunk_schedule: whole waves, 1, 2, 3 ... up to HOST_CHUNK, no tiny tail"""
    out = []
    maxc = max(wave, HOST_CHUNK // wave * wave)
    off, nxt = 0, wave
    while off < n:
        left = n - off
        cc = min(nxt, left)
        rest = left - cc
        if 0 < rest < wave:
            cc = (left - wave) // wave * wave if left >= 2 * wave else left
        elif rest == 0 and left > 2 * wave:
            cc = (left - wave) // wave * wave
        out.append((off, cc))
        off += cc
        nxt = min(nxt + wave, maxc)
    return out


def dev_chunks(n):
    return [(lo, min(DEV_CHUNK, n - lo)) for lo in range(0, n, DEV_CHUNK)]


LAYOUTS = ("slice0", "ends", "third", "run", "all")


def layout_mask(kind, n, chunks, tfun):
    """positions of the marked (identity / refused) elements: the whole slice of thread 0, the first and last element of a
    few slices, every third element, one contiguous run of 2T, the whole batch"""
    mask = np.zeros(n, bool)
    for off, cnt in chunks:
        T = tfun(cnt)
        idx = np.arange(cnt)
        if kind == "slice0":
            mask[off + idx[idx % T == 0]] = True
        elif kind == "ends":
            live = min(T, cnt)
            for t in sorted({1, 2, 5, live // 3, live // 2, live - 2, live - 1}):
                if 0 <= t < cnt:
                    mask[off + t] = True
                    mask[off + t + (cnt - 1 - t) // T * T] = True
        elif kind == "third":
            mask[off + idx[idx % 3 == 0]] = True
        elif kind == "run":
            a = min(T // 3 + 1, cnt - 1)
            mask[off + a:off + min(cnt, a + 2 * T)] = True
        elif kind == "all":
            mask[off:off + cnt] = True
        elif kind == "mixed":   # the ECDSA layouts: slice 0, heads and tails of every 7th slice, one run of T/4
            mask[off + idx[idx % T == 0]] = True
            live = min(T, cnt)
            for t in range(1, live, 7):
                mask[off + t] = True
                mask[off + t + (cnt - 1 - t) // T * T] = True
            a = min(T // 3 + 1, cnt - 1)
            mask[off + a:off + min(cnt, a + T // 4)] = True
        else:
            raise ValueError(kind)
    return mask


def occupancy(n, chunks, tfun, mask):
    """(fewest, most elements per thread, slices with a marked element and another element, slices mixing marked and
    unmarked elements)"""
    lo, hi, shared, mixed = None, 0, 0, 0
    for off, cnt in chunks:
        T = tfun(cnt)
        sl = np.arange(cnt) % T
        size = np.bincount(sl, minlength=min(T, cnt))
        marked = np.bincount(sl, weights=mask[off:off + cnt].astype(np.int64), minlength=min(T, cnt))
        size, marked = size[:min(T, cnt)], marked[:min(T, cnt)]
        lo = int(size.min()) if lo is None else min(lo, int(size.min()))
        hi = max(hi, int(size.max()))
        shared += int(((size >= 2) & (marked >= 1)).sum())
        mixed += int(((marked >= 1) & (marked < size)).sum())
    return lo, hi, shared, mixed


def _report(kernel, name, mode, n, chunks, tfun, mask):
    lo, hi, shared, mixed = occupancy(n, chunks, tfun, mask)
    print(f"[occupancy] {kernel} {name} {mode} n={n} chunks={len(chunks)} elements/thread {lo}..{hi} "
          f"slices with a marked element and a neighbour {shared}, of them mixed {mixed}")
    return lo, hi, shared, mixed


def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def norm_tile(name, count=64, seed=3):
    """count distinct points with random Z as Jacobian and homogeneous records, the affine records they stand for, and
    identity records (Z = 0, arbitrary X, Y < p)"""
    c = _curve(name)
    p = c.p
    rng = random.Random(seed)
    ts = [rng.randrange(1, c.n) for _ in range(count)]
    xy, inf = ecref.mul_gen_batch(name, recs(c, ts), nthreads=NT)
    assert not inf.any()
    nb = _fb(c)
    xy = np.asarray(xy).reshape(count, 2 * nb)
    jac, hom, ident = [], [], []
    for i in range(count):
        x, y = pyref.dec_fe(c, xy[i, :nb].tobytes()), pyref.dec_fe(c, xy[i, nb:].tobytes())
        z = rng.randrange(1, p)
        jac.append(pyref.enc_fe(c, x * z * z % p) + pyref.enc_fe(c, y * z * z * z % p) + pyref.enc_fe(c, z))
        hom.append(pyref.enc_fe(c, x * z % p) + pyref.enc_fe(c, y * z % p) + pyref.enc_fe(c, z))
        ident.append(pyref.enc_fe(c, rng.randrange(p)) + pyref.enc_fe(c, rng.randrange(p)) + pyref.enc_fe(c, 0))
    arr = lambda rs: np.frombuffer(b"".join(rs), np.uint8).reshape(count, -1).copy()  # noqa: E731
    return arr(jac), arr(hom), arr(ident), xy.copy()


def _tiled(base, ident, mask):
    n = mask.size
    idx = np.arange(n) % base.shape[0]
    out = base[idx]
    out[mask] = ident[idx[mask]]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_normalize_slices_host_mode(engine, name):
    """batch_normalize / batch_normalize_hom at n = 2^18 through the host chunks, identities in each layout"""
    c = _curve(name)
    nb = _fb(c)
    n = 1 << 18
    sms = _sms()
    chunks = host_chunks(n, sms * per_sm(name))
    jac, hom, ident, exy = norm_tile(name)
    want_base = exy[np.arange(n) % 64]
    for kind in LAYOUTS:
        mask = layout_mask(kind, n, chunks, lambda m: norm_threads(m, sms))
        _report("normalize_kernel", name, f"host {kind}", n, chunks, lambda m: norm_threads(m, sms), mask)
        want = want_base.copy()
        want[mask] = 0
        for label, fn, base in (("jacobian", engine.batch_normalize, jac), ("homogeneous", engine.batch_normalize_hom, hom)):
            xy, inf = fn(name, _tiled(base, ident, mask))
            assert np.array_equal(inf.astype(bool), mask), f"{name} {label} {kind}: identity flags"
            bad = np.nonzero((np.asarray(xy).reshape(n, 2 * nb) != want).any(axis=1))[0]
            assert not bad.size, f"{name} {label} {kind}: {bad.size} wrong records, first at {bad[:8].tolist()}"


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_normalize_slices_device_pointers(name):
    """the same through device pointers, one launch over n = 33 (SMs x 256) + 5 elements: 31-32 per inversion"""
    import torch

    import ecgpu

    c = _curve(name)
    nb = _fb(c)
    sms = _sms()
    n = 33 * sms * 256 + 5
    chunks = dev_chunks(n)
    dev = torch.device("cuda:0")
    jac, hom, ident, exy = norm_tile(name, seed=4)
    idx = torch.arange(n, device=dev) % 64
    E = torch.from_numpy(exy).to(dev)[idx]
    ID = torch.from_numpy(ident).to(dev)
    eng = ecgpu.Engine([0], device_ptrs=True)
    try:
        eng.set_stream(torch.cuda.current_stream().cuda_stream)
        out = torch.empty(n * 2 * nb, dtype=torch.uint8, device=dev)
        oinf = torch.empty(n, dtype=torch.uint8, device=dev)
        for kind in LAYOUTS:
            mask_np = layout_mask(kind, n, chunks, lambda m: norm_threads(m, sms))
            _report("normalize_kernel", name, f"device {kind}", n, chunks, lambda m: norm_threads(m, sms), mask_np)
            mask = torch.from_numpy(mask_np).to(dev)
            want = E.clone()
            want[mask] = 0
            for label, fn, base in (("jacobian", eng.batch_normalize_ptr, jac), ("homogeneous", eng.batch_normalize_hom_ptr, hom)):
                X = torch.from_numpy(base).to(dev)[idx]
                X[mask] = ID[idx[mask]]
                out.fill_(0xAA)
                oinf.fill_(0xAA)
                fn(name, n, X.data_ptr(), out.data_ptr(), oinf.data_ptr())
                torch.cuda.synchronize()
                assert torch.equal(oinf.bool(), mask) and int(oinf.max()) <= 1, f"{name} {label} {kind}: identity flags"
                bad = torch.nonzero((out.view(n, 2 * nb) != want).any(dim=1)).flatten()
                assert bad.numel() == 0, f"{name} {label} {kind}: {bad.numel()} wrong records, first at {bad[:8].tolist()}"
                del X
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_x_only_normalize_slices(name):
    """mul_batch_x (normalize_kernel<F, true>) over n = 2 (SMs x 256) + 7 elements, two to three per thread: k = 0 and
    P = O in each layout, 64 distinct pairs elsewhere"""
    import torch

    import ecgpu

    c = _curve(name)
    nb = _fb(c)
    sms = _sms()
    n = 2 * sms * 256 + 7
    chunks = dev_chunks(n)
    rng = random.Random(9)
    ks = [rng.randrange(1, c.n) for _ in range(64)]
    Ps = [pyref.mul(c, rng.randrange(1, c.n), pyref.G(c)) for _ in range(4)]
    Ps = [Ps[i % 4] for i in range(64)]
    K64, (P64, _) = recs(c, ks).reshape(64, nb), pts(c, Ps)
    P64 = P64.reshape(64, 2 * nb)
    rxy, rinf = ecref.mul_batch(name, K64, P64, None, nthreads=NT)
    assert not rinf.any()
    ex = np.asarray(rxy).reshape(64, 2 * nb)[:, :nb]
    dev = torch.device("cuda:0")
    eng = ecgpu.Engine([0], device_ptrs=True)
    try:
        eng.set_stream(torch.cuda.current_stream().cuda_stream)
        for kind in LAYOUTS:
            mask = layout_mask(kind, n, chunks, lambda m: norm_threads(m, sms))
            _report("normalize_kernel<x-only>", name, f"device {kind}", n, chunks, lambda m: norm_threads(m, sms), mask)
            idx = np.arange(n) % 64
            K, P, I = K64[idx], P64[idx], np.zeros(n, np.uint8)
            marked = np.nonzero(mask)[0]
            K[marked[0::2]] = 0              # k = 0
            P[marked[1::2]] = 0              # P = O
            I[marked[1::2]] = 1
            want = ex[idx]
            want[mask] = 0
            kd, pd, idd = (torch.from_numpy(a).to(dev) for a in (K, P, I))
            out = torch.full((n * nb,), 0xAA, dtype=torch.uint8, device=dev)
            oinf = torch.full((n,), 0xAA, dtype=torch.uint8, device=dev)
            eng.mul_batch_x_ptr(name, n, kd.data_ptr(), pd.data_ptr(), idd.data_ptr(), out.data_ptr(), oinf.data_ptr())
            torch.cuda.synchronize()
            assert np.array_equal(oinf.cpu().numpy().astype(bool), mask), f"{name} {kind}: identity flags"
            bad = np.nonzero((out.cpu().numpy().reshape(n, nb) != want).any(axis=1))[0]
            assert not bad.size, f"{name} x-only {kind}: {bad.size} wrong, first at {bad[:8].tolist()}"
    finally:
        eng.close()


# ---- ECDSA front ends ----

def sign_tile(name, count=64, seed=11, low_s=False):
    """count signatures (z, r, s, Q, recid, d) made with the model's signing equation over points from the C restatement
    (pyref.ecdsa_sign computes the same; a sample is checked against it without a GPU)"""
    c = _curve(name)
    n, nb = c.n, _fb(c)
    rng = random.Random(seed)
    ds = [rng.randrange(1, n) for _ in range(count)]
    ks = [rng.randrange(1, n) for _ in range(count)]
    qxy, _ = ecref.mul_gen_batch(name, recs(c, ds), nthreads=NT)
    rxy, _ = ecref.mul_gen_batch(name, recs(c, ks), nthreads=NT)
    qxy, rxy = np.asarray(qxy).reshape(count, 2 * nb), np.asarray(rxy).reshape(count, 2 * nb)
    out = []
    for i in range(count):
        Rx, Ry = pyref.dec_fe(c, rxy[i, :nb].tobytes()), pyref.dec_fe(c, rxy[i, nb:].tobytes())
        Q = (pyref.dec_fe(c, qxy[i, :nb].tobytes()), pyref.dec_fe(c, qxy[i, nb:].tobytes()))
        z = rng.randrange(1 << (8 * nb)) if name != "p521" else rng.randrange(1 << 521)
        r = Rx % n
        s = pow(ks[i], -1, n) * (z + r * ds[i]) % n
        assert r and s
        rid = (Ry & 1) | (2 if Rx >= n else 0)
        if low_s and s > n // 2:
            s, rid = n - s, rid ^ 1
        out.append((z, r, s, Q, rid, ds[i], ks[i]))
    return out


REFUSALS = ("r=0", "s=0", "r=n", "s=n", "Q off curve", "Q coordinate >= p")


def ecdsa_variant(name, sig, kind):
    """(z, r, s, qx, qy) of one inserted entry and whether the front end must refuse it"""
    c = _curve(name)
    n, p, nb = c.n, c.p, _fb(c)
    z, r, s, Q, *_ = sig
    qx, qy = Q
    if kind == "r=0":
        r = 0
    elif kind == "s=0":
        s = 0
    elif kind == "r=n":
        r = n
    elif kind == "s=n":
        s = n
    elif kind == "Q off curve":
        qy = (qy + 1) % p
    elif kind == "Q coordinate >= p":
        if qy + p < 1 << (8 * nb):
            qy += p            # the same residue: a kernel that reduced instead of refusing would accept it
        elif qx + p < 1 << (8 * nb):
            qx += p
        else:
            qx = p
    elif kind == "high s":
        s = n - s
    elif kind == "z flipped":
        z ^= 1
    else:
        raise ValueError(kind)
    return z, r, s, qx, qy


def ecdsa_kinds(name):
    return REFUSALS + (("high s",) if name == "k256" else ()) + ("z flipped",)


def _rec(c, v, nb):
    return v.to_bytes(nb, pyref.byteorder(c))


def ecdsa_batch(name, n, mask, sigs):
    """records of a batch: the tile of signatures, the inserted kinds cycled over the marked positions"""
    c = _curve(name)
    nb = _fb(c)
    kinds = ecdsa_kinds(name)
    base = [(s[0], s[1], s[2], s[3][0], s[3][1]) for s in sigs]
    var = {k: [ecdsa_variant(name, s, k) for s in sigs] for k in kinds}

    def tab(rows):
        Z = np.frombuffer(b"".join(_rec(c, z, nb) for z, *_ in rows), np.uint8).reshape(len(rows), nb)
        S = np.frombuffer(b"".join(_rec(c, r, nb) + _rec(c, s, nb) for _, r, s, *_ in rows), np.uint8).reshape(len(rows), 2 * nb)
        Q = np.frombuffer(b"".join(_rec(c, x, nb) + _rec(c, y, nb) for *_, x, y in rows), np.uint8).reshape(len(rows), 2 * nb)
        return Z, S, Q

    m = len(sigs)
    idx = np.arange(n) % m
    Zb, Sb, Qb = tab(base)
    Z, S, Q = Zb[idx].copy(), Sb[idx].copy(), Qb[idx].copy()
    kind_at = np.full(n, -1, np.int64)
    marked = np.nonzero(mask)[0]
    for j, k in enumerate(kinds):
        at = marked[j::len(kinds)]
        kind_at[at] = j
        Zk, Sk, Qk = tab(var[k])
        Z[at], S[at], Q[at] = Zk[idx[at]], Sk[idx[at]], Qk[idx[at]]
    return Z, S, Q, kind_at


def _ecdsa_tile(name):
    return sign_tile(name, low_s=(name == "k256"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ECDSA_NAMES)
def test_ecdsa_front_end_slices(engine, name):
    """ecdsa_verify_batch over n = 3 (SMs x 128) + 7 signatures (three per front-end thread): refusals at slice heads,
    tails and in a run must not spoil the s^-1 of their neighbours; every untouched signature verifies"""
    sms = _sms()
    n = 3 * sms * 128 + 7
    chunks = host_chunks(n, sms * per_sm(name))
    tf = lambda m: prep_threads(m, sms)  # noqa: E731
    mask = layout_mask("mixed", n, chunks, tf)
    sigs = _ecdsa_tile(name)
    Z, S, Q, kind_at = ecdsa_batch(name, n, mask, sigs)
    kinds = ecdsa_kinds(name)
    refused = (kind_at >= 0) & (kind_at < len(REFUSALS) + (1 if name == "k256" else 0))
    _report("ecdsa_prep_kernel" if name in ("k256", "p256") else "ecdsa_prep_generic_kernel", name, "host mixed", n, chunks, tf, refused)
    valid = engine.ecdsa_verify_batch(name, Z.reshape(-1), S.reshape(-1), Q.reshape(-1), low_s_only=(name == "k256"))
    want = kind_at < 0
    bad = np.nonzero(valid.astype(bool) != want)[0]
    assert not bad.size, (f"{name}: {bad.size} wrong verdicts, first "
                          f"{[(int(i), kinds[kind_at[i]] if kind_at[i] >= 0 else 'untouched', int(i) % tf(n)) for i in bad[:8]]}")
    assert valid.sum() == (~mask).sum()


def recovery_nonresidues(name, count, seed=13):
    """x < n for which x^3 + a x + b has no square root mod p"""
    c = _curve(name)
    rng = random.Random(seed)
    out = []
    while len(out) < count:
        x = rng.randrange(1, c.n)
        if pow((x * x * x + c.a * x + c.b) % c.p, (c.p - 1) // 2, c.p) == c.p - 1:
            out.append(x)
    return out


RECOVER_KINDS = ("recid=4", "recid=255", "r=n", "r=n+1", "r+n>=p", "x not a residue", "r=0", "s=0")


def recover_variant(name, sig, kind, nonres):
    c = _curve(name)
    n, p = c.n, c.p
    z, r, s, Q, rid, *_ = sig
    if kind == "recid=4":
        rid = 4 + (rid & 3)
    elif kind == "recid=255":
        rid = 255
    elif kind == "r=n":
        r = n
    elif kind == "r=n+1":
        r = n + 1
    elif kind == "r+n>=p":
        assert r + n >= p
        rid |= 2
    elif kind == "x not a residue":
        r, rid = nonres, rid & 1
    elif kind == "r=0":
        r = 0
    elif kind == "s=0":
        s = 0
    return z, r, s, rid


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["k256", "p256"])
def test_ecdsa_recover_front_end_slices(engine, name):
    """ecdsa_recover_batch in the same layouts: refused entries give 64 zero bytes and valid = 0, every untouched entry
    its signer's key"""
    c = _curve(name)
    sms = _sms()
    n = 3 * sms * 128 + 7
    chunks = host_chunks(n, sms * per_sm(name))
    tf = lambda m: prep_threads(m, sms)  # noqa: E731
    mask = layout_mask("mixed", n, chunks, tf)
    _report("ecdsa_recover_prep_kernel", name, "host mixed", n, chunks, tf, mask)
    low = name == "k256"
    sigs = [s for s in sign_tile(name, seed=21, low_s=low) if s[1] + c.n >= c.p]
    nonres = recovery_nonresidues(name, len(sigs))
    m = len(sigs)
    idx = np.arange(n) % m

    def tab(rows):
        Z = np.frombuffer(b"".join(z.to_bytes(32, "big") for z, *_ in rows), np.uint8).reshape(m, 32)
        S = np.frombuffer(b"".join(r.to_bytes(32, "big") + s.to_bytes(32, "big") for _, r, s, _ in rows), np.uint8).reshape(m, 64)
        R = np.array([rid for *_, rid in rows], np.uint8)
        return Z, S, R

    Zb, Sb, Rb = tab([(s[0], s[1], s[2], s[4]) for s in sigs])
    Qb = np.frombuffer(b"".join(s[3][0].to_bytes(32, "big") + s[3][1].to_bytes(32, "big") for s in sigs), np.uint8).reshape(m, 64)
    Z, S, R = Zb[idx].copy(), Sb[idx].copy(), Rb[idx].copy()
    kind_at = np.full(n, -1, np.int64)
    marked = np.nonzero(mask)[0]
    for j, k in enumerate(RECOVER_KINDS):
        at = marked[j::len(RECOVER_KINDS)]
        kind_at[at] = j
        Zk, Sk, Rk = tab([recover_variant(name, s, k, nonres[i]) for i, s in enumerate(sigs)])
        Z[at], S[at], R[at] = Zk[idx[at]], Sk[idx[at]], Rk[idx[at]]
    xy, valid = engine.ecdsa_recover_batch(name, Z.reshape(-1), S.reshape(-1), R, low_s_only=low)
    want_xy = Qb[idx].copy()
    want_xy[mask] = 0
    bad = np.nonzero((valid.astype(bool) != ~mask) | (np.asarray(xy).reshape(n, 64) != want_xy).any(axis=1))[0]
    assert not bad.size, (f"{name}: {bad.size} wrong, first "
                          f"{[(int(i), RECOVER_KINDS[kind_at[i]] if kind_at[i] >= 0 else 'untouched', int(i) % tf(n)) for i in bad[:8]]}")


# ---------------------------------------------------------------------------------------------------------------------
# C. bucket method with cancellation

MSM_N = (1 << 14) + 3


def condensed(name, ks, Ps):
    """the same sum with one term per distinct point (scalars added mod n): what the C restatement gets"""
    c = _curve(name)
    acc = {}
    for k, P in zip(ks, Ps):
        if P is not None:
            acc[P] = (acc.get(P, 0) + k) % c.n
    return list(acc.values()), list(acc.keys())


def bucket_inputs(name, seed=31):
    """{label: (scalars, points)} of MSM_N terms each"""
    c = _curve(name)
    n = c.n
    rng = random.Random(seed)
    ts = [rng.randrange(1, n) for _ in range(64)]
    nb = _fb(c)
    xy, _ = ecref.mul_gen_batch(name, recs(c, ts), nthreads=NT)
    xy = np.asarray(xy).reshape(64, 2 * nb)
    base = [(pyref.dec_fe(c, xy[i, :nb].tobytes()), pyref.dec_fe(c, xy[i, nb:].tobytes())) for i in range(64)]
    half = (MSM_N - 3) // 2
    out = {}
    ks, Ps = [], []
    for i in range(half):                      # k P + (n - k) P
        k = rng.randrange(1, n)
        ks += [k, n - k]
        Ps += [base[i % 64]] * 2
    ks += [0, rng.randrange(1, n), 0]
    Ps += [base[1], None, None]
    out["pairs"] = (ks, Ps)
    k64 = [rng.randrange(1, n) for _ in range(64)]  # 64 terms repeated: equal terms share a bucket in every window
    out["repeated"] = ([k64[i % 64] for i in range(MSM_N)], [base[i % 64] for i in range(MSM_N)])
    ks, Ps = [], []
    for i in range(half):                      # P and -P with equal digits
        k = rng.randrange(1, n)
        ks += [k, k]
        Ps += [base[i % 64], pyref.neg(c, base[i % 64])]
    ks += [rng.randrange(1, n) for _ in range(3)]
    Ps += [base[5], base[6], base[7]]
    out["P and -P"] = (ks, Ps)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_bucket_method_cancellation(engine, name):
    """lincomb and lincomb_partial + point_sum over 2^14 + 3 terms (the bucket method, below the skew refusal: the same
    number of kernel launches as a random input of that size) against ecref.lincomb"""
    c = _curve(name)
    nb = _fb(c)
    inputs = bucket_inputs(name)
    rng = random.Random(8)
    rk = recs(c, [rng.randrange(c.n) for _ in range(MSM_N)])
    rxy, rinf = pts(c, inputs["repeated"][1])
    l0 = engine.kernel_launches
    engine.lincomb(name, rk, rxy, rinf)
    bucket_launches = engine.kernel_launches - l0
    for label, (ks, Ps) in inputs.items():
        K = recs(c, ks)
        pxy, pinf = pts(c, Ps)
        ck, cP = condensed(name, ks, Ps)
        cxy, cinf = pts(c, cP)
        want = ecref.lincomb(name, recs(c, ck), cxy, cinf, nthreads=NT)
        if label == "pairs":
            assert want[1] == 1
        l0 = engine.kernel_launches
        got = engine.lincomb(name, K, pxy, pinf)
        assert engine.kernel_launches - l0 == bucket_launches, f"{name} {label}: not the bucket path alone"
        assert np.array_equal(got[0], want[0]) and got[1] == want[1], f"{name} {label}: lincomb"
        h = MSM_N // 2
        p1 = engine.lincomb_partial(name, K[:nb * h], pxy[:2 * nb * h], pinf[:h])
        p2 = engine.lincomb_partial(name, K[nb * h:], pxy[2 * nb * h:], pinf[h:])
        got = engine.point_sum(name, np.concatenate([p1, p2]))
        assert np.array_equal(got[0], want[0]) and got[1] == want[1], f"{name} {label}: lincomb_partial + point_sum"


# ---------------------------------------------------------------------------------------------------------------------
# the all-inlined P-384 fixed-base kernel (tests/dev/fe_dev.cu) over the window patterns

def _p384_pattern_scalars():
    """(k, window, value, family): the window patterns, then families near n that narrow down where the inlined kernel
    goes wrong: n - i, n - 2^e, and n - 1 with one 16-bit window cleared"""
    c = pyref.P384
    cases = fixedbase_patterns("p384")
    extra = [(k, -1, k, "small") for k in range(1, 33)] + [(c.n - i, -1, i, "n-i") for i in range(1, 33)]
    extra += [(c.n - (1 << e), -1, e, "n-2^e") for e in range(384)]
    extra += [((c.n - 1) & ~(0xFFFF << (16 * w)), w, 0, "n-1 window cleared") for w in range(24)]
    return [x for x in cases + extra if x[0] != 0]


def _p384_run(inlined):
    import test_gpu_field_layer as fl

    be = fl.Backend("device")
    c = pyref.P384
    cases = _p384_pattern_scalars()
    ks = [k for k, *_ in cases]
    reads = {}
    for k in ks:
        for point, mult in fl._fb_reads(k, c.n):
            reads[point] = mult % c.n
    order = sorted(reads)
    txy, tinf = ecref.mul_gen_batch("p384", recs(c, [reads[i] for i in order]), nthreads=NT)
    assert not tinf.any()
    txy = np.asarray(txy).reshape(-1, 96)
    table = np.zeros((fl.FB_WINDOWS * fl.FB_ENTRIES + 1, 24), np.uint32)
    for j, point in enumerate(order):
        x, y = txy[j, :48].tobytes()[::-1], txy[j, 48:].tobytes()[::-1]   # big-endian records -> little-endian words
        table[point] = np.frombuffer(x + y, np.uint32)
    K = recs(c, ks)
    out = np.empty(36 * len(ks), np.uint32)
    st = np.zeros(2, np.uint32)
    be.ok(be.lib.dev_fixedbase_p384(inlined, len(ks), fl._p(K, fl.U8P), fl._p(table.reshape(-1)), fl._p(out), fl._p(st)))
    assert st[0] == 0
    got = fl._unpack_jac(fl._variants()[4], out)
    wxy, _ = ecref.mul_gen_batch("p384", K, nthreads=NT)
    wxy = np.asarray(wxy).reshape(-1, 96)
    want = [(int.from_bytes(wxy[i, :48].tobytes(), "big"), int.from_bytes(wxy[i, 48:].tobytes(), "big")) for i in range(len(ks))]
    bad = [cases[i][1:] for i in range(len(ks)) if got[i] != want[i]]
    return bad, len(ks)


@pytest.mark.gpu
def test_p384_fixedbase_call_based_window_patterns():
    """fixedbase_kernel<CurveP384> (what P-384 k*G runs) over every window pattern on a sparse table"""
    bad, total = _p384_run(0)
    assert not bad, f"{len(bad)}/{total} wrong: {bad[:12]}"


@pytest.mark.gpu
@pytest.mark.xfail(strict=True, reason="fixedbase_kernel<CurveP384I> built by nvcc 12.9 for sm_90a returns wrong points "
                                       "(DESIGN.md section 4); P-384 k*G uses the call-based field instead")
def test_p384_fixedbase_all_inlined_window_patterns():
    bad, total = _p384_run(1)
    fams = {}
    for w, v, f in bad:   # window patterns: (window, value); n - 1 with a window cleared: the window; others: i or e
        fams.setdefault(f, []).append((w, v) if f in ("0", "1", "r") else w if w >= 0 else v)
    print(f"[p384 inlined] {len(bad)}/{total} wrong; by family: {fams}")
    assert not bad, f"{len(bad)}/{total} wrong: {fams}"


# ---------------------------------------------------------------------------------------------------------------------
# without a GPU: the case builders and verdict rules

@pytest.mark.parametrize("name", NAMES)
def test_scalar_sets_stay_below_n_and_reach_the_endings(name):
    c = _curve(name)
    n, bl, nb = c.n, c.n.bit_length(), _fb(c)
    ks = scalar_set(name)
    assert all(0 <= k < n for k in ks) and len(ks) == len(set(ks))
    assert set(range(1024)) <= set(ks) and {n - i for i in range(1, 1024)} <= set(ks)
    assert {n - (1 << e) for e in range(bl)} <= set(ks)
    assert 2000 < len(ks) < 7000
    K = recs(c, ks)
    assert K.size == nb * len(ks)
    assert pyref.dec_fe(c, K[nb:2 * nb].tobytes()) == ks[1]          # the curve's byte order (bign: little-endian)
    if name == "k256":
        assert (3 * K256_LAMBDA + 1) % n in ks and (n - 40 * K256_LAMBDA - 2) % n in ks
    pats = fixedbase_patterns(name)
    windows = {w for _, w, _, _ in pats}
    assert len(windows) == {"p224": 14, "p521": 33, "p192": 12, "p384": 24, "bp384r1": 24, "bp384t1": 24}.get(name, 16)
    assert all(0 <= k < n for k, *_ in pats)
    top = max(windows)
    # the top window's all-ones pattern fills exactly the bits below the length of n (P-521: 9 bits)
    assert max(v for _, w, v, _ in pats if w == top) == (1 << (bl - 16 * top)) - 1


@pytest.mark.parametrize("name", ["k256", "p224", "bignp256", "p521"])
def test_mul_gen_add_cases_end_where_stated(name):
    c = _curve(name)
    cases = mul_gen_add_cases(name, count=4)
    want, _ = _model_sum(name, cases)
    G = pyref.G(c)
    for (a, b, P, kind), w in zip(cases, want):
        if kind == "identity":
            assert w is None
        elif kind == "double":
            aG = pyref.mul(c, a, G)
            assert w == pyref.add(c, aG, aG)
        elif kind == "a*G":
            assert w == pyref.mul(c, a, G)
        else:
            assert w == pyref.mul(c, b, P)


def test_slice_mirrors():
    """the mirrors of the launch geometry on a 132-SM device: slice sizes, chunk schedule, layouts"""
    sms = 132
    assert norm_threads(1 << 18, sms) == 33792 and prep_threads(3 * sms * 128 + 7, sms) == 16896
    n = 33 * sms * 256 + 5
    T = norm_threads(n, sms)
    assert n // T >= 31 and -(-n // T) <= 33
    for wave in (33792, 50688, 67584, 84480):
        ch = host_chunks(1 << 18, wave)
        assert sum(cc for _, cc in ch) == 1 << 18 and all(o == sum(cc for _, cc in ch[:i]) for i, (o, _) in enumerate(ch))
        assert all(cc <= max(wave, HOST_CHUNK // wave * wave) for _, cc in ch)
    assert host_chunks(3 * sms * 128 + 7, 132 * 384) == [(0, 3 * sms * 128 + 7)]
    ch = [(0, n)]
    tf = lambda m: norm_threads(m, sms)  # noqa: E731
    m0 = layout_mask("slice0", n, ch, tf)
    assert m0.sum() == -(-n // T) and m0[0] and m0[T] and not m0[1]
    ends = layout_mask("ends", n, ch, tf)
    assert ends[1] and ends[1 + (n - 2) // T * T] and not ends[1 + T]
    run = layout_mask("run", n, ch, tf)
    assert run.sum() == 2 * T
    lo, hi, shared, mixed = occupancy(n, ch, tf, layout_mask("mixed", n, ch, tf))
    assert lo >= 31 and hi <= 33 and shared > T // 8 and mixed > T // 8
    assert occupancy(n, ch, tf, layout_mask("all", n, ch, tf))[3] == 0


@pytest.mark.parametrize("name", ["k256", "p256", "p224", "bp384t1", "p521"])
def test_ecdsa_cases_against_the_model(name):
    """a sample of the tile and of every inserted kind against pyref.ecdsa_sign / ecdsa_verify"""
    c = _curve(name)
    low = name == "k256"
    sigs = sign_tile(name, count=3, low_s=low)
    for z, r, s, Q, rid, d, k in sigs[:2]:
        rr, ss = pyref.ecdsa_sign(c, d, z % c.n, k)
        assert rr == r and ss in (s, c.n - s)
        assert pyref.ecdsa_verify(c, z, r, s, Q, low_s_only=low)
    for kind in ecdsa_kinds(name):   # every inserted entry fails: the refusals in the front end, a flipped z at the end
        z, r, s, qx, qy = ecdsa_variant(name, sigs[0], kind)
        assert not pyref.ecdsa_verify(c, z, r, s, (qx, qy), low_s_only=low), kind
    # the inserted records land where the layout says, kinds in turn
    n = 200
    mask = np.zeros(n, bool)
    mask[[0, 7, 50, 51, 52, 199]] = True
    Z, S, Q, kind_at = ecdsa_batch(name, n, mask, sigs)
    assert (kind_at >= 0).sum() == 6 and np.array_equal(kind_at >= 0, mask)
    nb = _fb(c)
    assert np.array_equal(S[1], S[1 + 3 * 10]) and not np.array_equal(S[0], S[3])


@pytest.mark.parametrize("name", ["k256", "p256"])
def test_recovery_cases_against_the_model(name):
    c = _curve(name)
    low = name == "k256"
    sigs = [s for s in sign_tile(name, count=4, seed=21, low_s=low) if s[1] + c.n >= c.p]
    assert sigs
    nonres = recovery_nonresidues(name, 2)
    z, r, s, Q, rid, *_ = sigs[0]
    assert pyref.ecdsa_recover(c, z, r, s, rid, low) == Q
    for kind in RECOVER_KINDS:
        zz, rr, ss, rd = recover_variant(name, sigs[0], kind, nonres[0])
        assert rr < 1 << 256 and rd < 256
        assert pyref.ecdsa_recover(c, zz, rr, ss, rd, low) is None, kind


@pytest.mark.parametrize("name", ["k256", "p384", "p521"])
def test_bucket_inputs_sum_as_stated(name):
    c = _curve(name)
    inputs = bucket_inputs(name)
    for label, (ks, Ps) in inputs.items():
        assert len(ks) == len(Ps) == MSM_N
        ck, cP = condensed(name, ks, Ps)
        terms = dict(zip(cP, ck))
        if label == "pairs":
            assert not any(ck)
        elif label == "repeated":
            assert len(cP) == 64 and all(terms[P] == k * math.ceil((MSM_N - i) / 64) % c.n for i, (k, P) in enumerate(zip(ks[:64], Ps[:64])))
        else:
            # P and -P carry equal scalars, so only the three closing terms remain
            extra = dict(zip(Ps[-3:], ks[-3:]))
            for P in terms:
                Pn = pyref.neg(c, P)
                assert (terms[P] - terms.get(Pn, 0)) % c.n == (extra.get(P, 0) - extra.get(Pn, 0)) % c.n
