"""The field and point layers as the kernels compile them (tests/dev/fe_dev.cu), against Python integers.

Every field policy a production kernel instantiates — the call-based and the all-inlined hand-written fields of
secp256k1, P-256 and P-384, the nine Montgomery curve fields and the twelve scalar fields — runs every operation on raw
limbs under each production launch bound.  Nothing is range-checked or converted on the way in, so the weakly reduced
inputs in [p, 2^(32 NL)) that the hand-written fields accept reach the arithmetic, and the raw result is checked for its
congruence and its documented range.  The point chains mirror fixedbase_accumulate (mixed additions with conditional
negation, a selected last step) and steer into the exceptional branches: P = Q, P = -Q, an identity accumulator.

The device build (libecgdev.so) runs under the `gpu` marker; the same bodies compiled for the host (libecgdevsim.so, C
emulation of the carry primitives) run everywhere, so the generators and expected values are exercised without a GPU."""
import ctypes
import os
import random

import numpy as np
import pytest

import pyref

DEV = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dev")
U32P = ctypes.POINTER(ctypes.c_uint32)
U8P = ctypes.POINTER(ctypes.c_uint8)
OPS = {"add": 0, "sub": 1, "mul": 2, "sqr": 3, "neg": 4, "half": 5, "mul3": 6, "inv": 7, "normalize": 8, "mul8": 9, "is_zero": 10}
SHAPES = ("(256)", "(128, 4)", "(256, 2)", "(128, 3)", "(128, 5)")


class Backend:
    def __init__(self, kind):
        import __graft_entry__ as ge

        ge.build()
        self.kind = kind
        self.lib = ctypes.CDLL(os.path.join(DEV, "libecgdev.so" if kind == "device" else "libecgdevsim.so"))
        L = self.lib
        L.dev_fe_op.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_size_t, U32P, U32P, U32P, U32P]
        L.dev_madd_chain.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_int, U32P, U32P, U8P, U8P, U32P]
        L.dev_jac_op.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_size_t, U32P, U32P, U32P]
        L.dev_fixedbase_p384.argtypes = [ctypes.c_int, ctypes.c_size_t, U8P, U32P, U32P, U32P]
        L.dev_variant_info.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_char_p)] + [ctypes.POINTER(ctypes.c_int)] * 4
        L.dev_error_string.restype = ctypes.c_char_p
        assert L.dev_is_device() == (1 if kind == "device" else 0)
        # the host build has no launch shapes: one run stands for all
        self.shapes = range(L.dev_shape_count()) if kind == "device" else range(1)
        # elements per operation (inversions are ~400 multiplications each)
        self.n, self.n_inv, self.n_pts = (1 << 14, 1 << 10, 1 << 11) if kind == "device" else (1 << 10, 24, 96)

    def ok(self, rc):
        assert rc == 0, f"rc {rc}: {self.lib.dev_error_string(rc).decode()}"


@pytest.fixture(scope="module", params=[pytest.param("host", id="host"), pytest.param("device", id="device", marks=pytest.mark.gpu)])
def be(request):
    return Backend(request.param)


def _p(a, t=U32P):
    return a.ctypes.data_as(t)


class Variant:
    """A field policy of fe_dev.cu: its modulus, limb count and internal form, and the curve it serves (if any)."""

    def __init__(self, vid):
        name, nl, mont, weak, amode = ctypes.c_char_p(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        lib = ctypes.CDLL(os.path.join(DEV, "libecgdevsim.so"))
        lib.dev_variant_info.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_char_p)] + [ctypes.POINTER(ctypes.c_int)] * 4
        assert lib.dev_variant_info(vid, ctypes.byref(name), ctypes.byref(nl), ctypes.byref(mont), ctypes.byref(weak), ctypes.byref(amode)) == 0
        self.id, self.name, self.nl, self.mont, self.weak, self.amode = vid, name.value.decode(), nl.value, bool(mont.value), bool(weak.value), amode.value
        base = self.name[2:] if self.name.startswith("n_") else self.name.replace("_inl", "")
        self.curve = pyref.CURVES[base]
        self.m = self.curve.n if self.name.startswith("n_") else self.curve.p
        self.W = 1 << (32 * self.nl)
        self.R = self.W % self.m if self.mont else 1
        self.Rinv = pow(self.R, -1, self.m)

    # raw limbs <-> integers
    def pack(self, vals):
        return np.frombuffer(b"".join(v.to_bytes(4 * self.nl, "little") for v in vals), np.uint32).copy()

    def unpack(self, arr):
        b = np.ascontiguousarray(arr).view(np.uint8).reshape(-1, 4 * self.nl)
        return [int.from_bytes(r.tobytes(), "little") for r in b]

    def enc(self, v, rng=None):
        """internal form of the field value v; a weakly reduced field sometimes gets the representative v R + m"""
        r = v * self.R % self.m
        if self.weak and rng is not None and r + self.m < self.W and rng.random() < 0.3:
            r += self.m
        return r

    def dec(self, r):
        return r * self.Rinv % self.m

    def edges(self):
        """0, 1, p - 1, p, p + 1, 2^(32 NL) - 1, 2^(32 NL) - p, ... (the values at or above p only where the policy takes
        them), and bit patterns around the top of the modulus and the P-521 fold / rotation boundaries"""
        m, W = self.m, self.W
        top = 1 << (m.bit_length() - 1)
        edges = [0, 1, 2, m - 1, m - 2, (m + 1) // 2, (m - 1) // 2, top, top - 1, (1 << 23) - 1, m - (1 << 23), W // 2 % m]
        if self.weak:
            edges += [m, m + 1, m + 2, W - 1, W - 2, W - m, W - m - 1, W - m + 1, 2 * m - W if 2 * m > W else 0]
        return sorted(set(e for e in edges if 0 <= e < (W if self.weak else m)))

    def inputs(self, n, rng):
        """every ordered pair of edge values first, then limb patterns and uniform values"""
        m, W, nl = self.m, self.W, self.nl
        edges = self.edges()
        pairs = [(x, y) for x in edges for y in edges]
        a, b = self._fill(n - len(pairs), rng), self._fill(n - len(pairs), rng)
        # the edges themselves lead (the inversion runs on a prefix), the pairs close the batch
        return edges + a[len(edges):] + [x for x, _ in pairs], edges[::-1] + b[len(edges):] + [y for _, y in pairs]

    def _fill(self, n, rng):
        m, W, nl = self.m, self.W, self.nl
        limbs = [0, 1, 0xFFFFFFFF, 0xFFFFFFFE]
        pats = []
        for _ in range(n // 4):
            v = sum((rng.choice(limbs) if rng.random() < 0.8 else rng.getrandbits(32)) << (32 * i) for i in range(nl))
            pats.append(v if self.weak or v < m else v % m)
        hi = W if self.weak else m
        vals = pats
        while len(vals) < n:
            vals.append(rng.randrange(hi))
        vals = vals[:n]
        rng.shuffle(vals)
        return vals

    def expect(self, op, a, b):
        m = self.m
        if op == "add":
            return (a + b) % m
        if op == "sub":
            return (a - b) % m
        if op == "mul":
            return a * b * self.Rinv % m
        if op == "sqr":
            return a * a * self.Rinv % m
        if op == "neg":
            return -a % m
        if op == "half":
            return a * pow(2, -1, m) % m
        if op == "mul3":
            return 3 * a % m
        if op == "mul8":
            return 8 * a % m
        if op == "inv":  # a^(p-2) in the policy's own arithmetic: (R^2 / a) in the Montgomery form
            return 0 if a % m == 0 else self.R * self.R * pow(a, -1, m) % m
        if op == "normalize":
            return a % m
        raise ValueError(op)


VARIANTS = [Variant(v) for v in range(27)] if os.path.exists(os.path.join(DEV, "libecgdevsim.so")) else []


def _variants():
    if not VARIANTS:  # collected before build(): build now
        import __graft_entry__ as ge

        ge.build()
        VARIANTS.extend(Variant(v) for v in range(27))
    return VARIANTS


def _fe_run(be, v, op, shape, A, B):
    n = len(A) // v.nl
    raw, norm = np.empty_like(A), np.empty_like(A)
    be.ok(be.lib.dev_fe_op(v.id, shape, OPS[op], n, _p(A), _p(B), _p(raw), _p(norm)))
    return raw, norm


def _check_fe(v, op, a, b, raw, norm, shape):
    R, N = v.unpack(raw), v.unpack(norm)
    for i, (x, y, r, q) in enumerate(zip(a, b, R, N)):
        where = f"{v.name} {op} shape {SHAPES[shape]} a={x:#x} b={y:#x}"
        if op == "is_zero":
            assert r == q == (1 if x % v.m == 0 else 0), where
            continue
        want = v.expect(op, x, y)
        assert r % v.m == want, f"{where}: raw {r:#x} is not congruent to {want:#x}"
        assert r < (v.W if v.weak else v.m), f"{where}: raw {r:#x} out of range"
        assert q == want, f"{where}: normalized {q:#x} != {want:#x}"


@pytest.mark.parametrize("vid", range(27), ids=lambda i: _variants()[i].name)
def test_field_ops_every_policy_and_shape(be, vid):
    v = _variants()[vid]
    rng = random.Random(1000 + vid)
    a, b = v.inputs(be.n, rng)
    A, B = v.pack(a), v.pack(b)
    for op in OPS:
        n = be.n_inv if op == "inv" else be.n
        An, Bn = A[: n * v.nl], B[: n * v.nl]
        ref = None
        for shape in be.shapes:
            raw, norm = _fe_run(be, v, op, shape, An, Bn)
            if ref is None:
                _check_fe(v, op, a[:n], b[:n], raw, norm, shape)
                ref = (raw, norm)
            elif not (np.array_equal(raw, ref[0]) and np.array_equal(norm, ref[1])):
                _check_fe(v, op, a[:n], b[:n], raw, norm, shape)  # names the element and the kind of error
                pytest.fail(f"{v.name} {op}: shape {SHAPES[shape]} differs from {SHAPES[0]} bit for bit")


# ---- points ---------------------------------------------------------------------------------------------------------

POINT_VARIANTS = [i for i in range(15)]


def _pool(c, rng, count):
    """distinct random points: a few scalar multiples of G, then sums of earlier ones"""
    pool = [pyref.mul(c, rng.randrange(1, c.n), pyref.G(c)) for _ in range(4)]
    while len(pool) < count:
        P = pyref.add(c, pool[-1], rng.choice(pool))
        if P is not None:
            pool.append(P)
    return pool


def _jac(v, P, rng, zero_z=False):
    """Jacobian internal-form encoding of affine P (None: the identity) with a random Z"""
    if P is None or zero_z:
        z0 = 0 if not v.weak or rng.random() < 0.5 else v.m  # Z = p is the identity too in a weakly reduced field
        return [v.enc(rng.randrange(1, v.m), rng), v.enc(rng.randrange(1, v.m), rng), z0]
    z = rng.randrange(1, v.m)
    return [v.enc(P[0] * z * z % v.m, rng), v.enc(P[1] * z ** 3 % v.m, rng), v.enc(z, rng)]


def _affine(v, X, Y, Z):
    X, Y, Z = v.dec(X), v.dec(Y), v.dec(Z)
    if Z == 0:
        return None
    zi = pow(Z, -1, v.m)
    return (X * zi * zi % v.m, Y * zi ** 3 % v.m)


def _unpack_jac(v, out):
    w = v.unpack(out)
    return [_affine(v, w[3 * i], w[3 * i + 1], w[3 * i + 2]) for i in range(len(w) // 3)]


@pytest.mark.parametrize("vid", POINT_VARIANTS, ids=lambda i: _variants()[i].name)
def test_madd_chain_exceptional_branches(be, vid):
    """fixedbase_accumulate's step sequence; chains of four kinds: random steps; a step that adds the accumulator to
    itself (P = Q: the doubling branch); a step that adds its negation (P = -Q: the identity) followed by steps from the
    identity accumulator; and a last step dropped by jac_csel"""
    v = _variants()[vid]
    c = v.curve
    rng = random.Random(2000 + vid)
    L = 6
    pool = _pool(c, rng, 48)
    n = be.n_pts
    starts, qs, negs, sels, want = [], [], [], [], []
    for i in range(n):
        kind = i % 4
        acc = rng.choice(pool)
        starts += [v.enc(acc[0], rng), v.enc(acc[1], rng)]
        sel = rng.randrange(2) if kind == 3 else 1
        for s in range(L):
            q = rng.choice(pool)
            neg = rng.randrange(2)
            if kind == 1 and s == 2 and acc is not None:
                q, neg = acc, 0                        # P = Q
            elif kind == 2 and s == 1 and acc is not None:
                q, neg = acc, 1                        # P = -Q: the accumulator becomes the identity
            elif kind == 1 and s == 4 and acc is not None:
                q, neg = pyref.neg(c, acc), 1          # P = Q again, through the negation flag
            qs += [v.enc(q[0], rng), v.enc(q[1], rng)]
            negs.append(neg)
            step = pyref.add(c, acc, pyref.neg(c, q) if neg else q)
            if s + 1 < L or sel:
                acc = step
        sels.append(sel)
        want.append(acc)
    S, Q = v.pack(starts), v.pack(qs)
    NG, SL = np.array(negs, np.uint8), np.array(sels, np.uint8)
    for shape in be.shapes:
        out = np.empty(3 * v.nl * n, np.uint32)
        be.ok(be.lib.dev_madd_chain(v.id, shape, n, L, _p(S), _p(Q), _p(NG, U8P), _p(SL, U8P), _p(out)))
        got = _unpack_jac(v, out)
        bad = [i for i in range(n) if got[i] != want[i]]
        assert not bad, f"{v.name} shape {SHAPES[shape]}: {len(bad)} wrong chains, first {bad[0]} (kind {bad[0] % 4})"


@pytest.mark.parametrize("vid", POINT_VARIANTS, ids=lambda i: _variants()[i].name)
def test_jac_dbl_add_madd_branches(be, vid):
    """jac_dbl / jac_add / jac_madd on random Z, with identity operands (Z = 0, and Z = p where that is a representable
    value), P = Q and P = -Q under different Z"""
    v = _variants()[vid]
    c = v.curve
    rng = random.Random(3000 + vid)
    pool = _pool(c, rng, 32)
    n = be.n_pts
    Ps, Qs, p_in, q_in = [], [], [], []
    for i in range(n):
        P = rng.choice(pool)
        kind = i % 6
        Q = {0: rng.choice(pool), 1: P, 2: pyref.neg(c, P), 3: None, 4: rng.choice(pool), 5: P}[kind]
        if kind == 4:
            P = None
        if kind == 5:
            P, Q = None, None
        Ps.append(P)
        Qs.append(Q)
        p_in += _jac(v, P, rng)
        q_in += _jac(v, Q, rng)
    PA, QA = v.pack(p_in), v.pack(q_in)
    # the mixed addition takes Q affine (Z = 1) and not the identity
    qa_in = []
    for Q in Qs:
        Qm = Q if Q is not None else pool[0]
        qa_in += [v.enc(Qm[0], rng), v.enc(Qm[1], rng), v.enc(1)]
    QM = v.pack(qa_in)
    want = {0: [pyref.add(c, P, P) for P in Ps],
            1: [pyref.add(c, P, Q) for P, Q in zip(Ps, Qs)],
            2: [pyref.add(c, P, Q if Q is not None else pool[0]) for P, Q in zip(Ps, Qs)]}
    for shape in be.shapes:
        for op, Qin in ((0, QA), (1, QA), (2, QM)):
            out = np.empty(3 * v.nl * n, np.uint32)
            be.ok(be.lib.dev_jac_op(v.id, shape, op, n, _p(PA), _p(Qin), _p(out)))
            got = _unpack_jac(v, out)
            bad = [i for i in range(n) if got[i] != want[op][i]]
            assert not bad, f"{v.name} {['dbl', 'add', 'madd'][op]} shape {SHAPES[shape]}: {len(bad)} wrong, first {bad[0]} (kind {bad[0] % 6})"


def test_scalar_fields_have_no_point_entries(be):
    v = _variants()[15]
    z = np.zeros(3 * v.nl, np.uint32)
    assert be.lib.dev_jac_op(v.id, 0, 0, 1, _p(z), _p(z), _p(z)) == -1
    assert be.lib.dev_fe_op(0, 5, 0, 1, _p(z), _p(z), _p(z), _p(z)) == -1  # no such launch shape


# ---- P-384 fixed-base kernel, call-based and all-inlined ------------------------------------------------------------

FB_W, FB_ENTRIES, FB_WINDOWS = 16, 1 << 15, 24


def _fb_reads(k, n):
    """(table point, value) pairs fixedbase_accumulate reads for scalar k (recode_full: m = k or k + 1, odd; 16-bit windows
    of m >> 1 select odd multiples (2 idx + 1) 2^(16 i) G; the top entry is 2^384 G; entry 0 = G corrects the parity)"""
    even = 1 - (k & 1)
    h = (k + even) >> 1
    reads = [(FB_WINDOWS * FB_ENTRIES, 1 << 384), (0, 1)]
    for i in range(FB_WINDOWS):
        w = (h >> (16 * i)) & 0xFFFF
        idx = (w & (FB_ENTRIES - 1)) if w >> 15 else (FB_ENTRIES - 1 - w)
        reads.append((i * FB_ENTRIES + idx, (2 * idx + 1) << (16 * i)))
    return reads


def _fixedbase_p384_case(be, inlined):
    """fixedbase_kernel<CurveP384I> (inlined: every field operation inlined under the kernel's (128, 4) bound) or
    fixedbase_kernel<CurveP384> over a sparse table holding only the entries these scalars read: the reference's P-384
    vectors (k = 1..20 and k near n), edges, random scalars"""
    if be.kind != "device":
        pytest.skip("a kernel launch")
    from helpers import golden

    c = pyref.P384
    g = golden("p384")
    ks = list(range(1, 21)) + [int(v["k"], 16) for v in g["group"]["mul"]] + [c.n - 1, c.n - 2, 2**383, 2**192 + 1, (c.n - 1) // 2]
    rng = random.Random(384)
    ks += [rng.randrange(c.n) for _ in range(24)]
    table = np.zeros(((FB_WINDOWS * FB_ENTRIES + 1), 24), np.uint32)
    done = set()
    for k in ks:
        for point, mult in _fb_reads(k, c.n):
            if point not in done:
                x, y = pyref.mul(c, mult, pyref.G(c))
                done.add(point)
                table[point] = np.frombuffer(x.to_bytes(48, "little") + y.to_bytes(48, "little"), np.uint32)
    K = np.frombuffer(b"".join(k.to_bytes(48, "big") for k in ks), np.uint8).copy()
    want = [pyref.mul(c, k, pyref.G(c)) for k in ks]
    out = np.empty(36 * len(ks), np.uint32)
    st = np.zeros(2, np.uint32)
    be.ok(be.lib.dev_fixedbase_p384(inlined, len(ks), _p(K, U8P), _p(table.reshape(-1)), _p(out), _p(st)))
    assert st[0] == 0
    got = _unpack_jac(_variants()[4], out)
    bad = [i for i in range(len(ks)) if got[i] != want[i]]
    assert not bad, f"{len(bad)}/{len(ks)} wrong, at {bad}"


@pytest.mark.gpu
def test_fixedbase_p384_call_based(be):
    """the kernel P-384 k*G runs (ecgpu.cu: FOR_CURVE_INL keeps CurveP384)"""
    _fixedbase_p384_case(be, 0)


@pytest.mark.gpu
@pytest.mark.xfail(strict=True, reason="fixedbase_kernel<CurveP384I> built by nvcc 12.9 for sm_90a returns wrong points for "
                                       "scalars near n among others (DESIGN.md section 4); P-384 k*G "
                                       "uses the call-based field instead")
def test_fixedbase_p384_all_inlined(be):
    _fixedbase_p384_case(be, 1)
