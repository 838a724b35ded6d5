"""Decaf448 (RFC 9496): the model (decaf448_model.py) against the reference's vectors and its own twisted formulas, the
device routines (tests/dev/decaf448_dev.cu: decode, encode, the variable-base and fixed-base kernels, the map,
expand_message_xof, the scalar transforms, the hash kernels, under the production launch bounds) against their host twin
and the model, and the ecg_decaf448_* entries through the C ABI, the Python and C++ mirrors.

Oracles: the reference's 16 multiples of G, its invalid records, its scalar_hash vector and the RFC 9497 DeriveKeyPair
vectors (tests/golden/decaf448.json, extracted by tools/extract_decaf448_golden.py), the reference's twisted formulas
restated in Python, and algebraic identities between the entries ([k]([a]G) == [k a]G, sum k_i [a_i]G == [sum k_i a_i]G,
[k]G == encode([-2k]B) through the Ed448 entry)."""
import ctypes
import json
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

import decaf448_model as D
import ed448_group_model as G
import ed448_model as M

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = os.path.join(HERE, "dev")
LIB = os.path.join(ROOT, "elliptic-curves_b200", "libecgpu.so")
GOLDEN = json.load(open(os.path.join(HERE, "golden", "decaf448.json")))
MULTS = [bytes.fromhex(h) for h in GOLDEN["multiples"]]
GEN = bytes.fromhex(GOLDEN["generator"])
U8P = ctypes.POINTER(ctypes.c_uint8)
U32P = ctypes.POINTER(ctypes.c_uint32)
U64P = ctypes.POINTER(ctypes.c_uint64)
P, L = M.P, M.L
ID = D.IDENTITY_BYTES
RO, NU = D.HASH_TO_CURVE_ID, D.ENCODE_TO_CURVE_ID


def enc_s(s: int) -> bytes:
    return s.to_bytes(56, "little")


def rand_point(rng):
    """a random valid encoding: [a]G for a random a"""
    return D.encode(M.mul(rng.randrange(L), D.G0))


def edge_records():
    """s = 0, 2, p - 1, p - 3, p + 1, 2^448 - 2, odd s, s >= p, and the reference's invalid records"""
    vals = [0, 1, 2, 3, P - 1, P - 2, P - 3, P, P + 1, P + 2, 2**448 - 2, 2**448 - 1]
    recs = [enc_s(v) for v in vals] + [bytes.fromhex(h) for h in GOLDEN["invalid"]] + MULTS
    return recs


def random_records(n, seed):
    rng = random.Random(seed)
    out = []
    for i in range(n):
        if i % 4 == 0:
            out.append(rng.getrandbits(448).to_bytes(56, "little"))  # mostly refused: odd or >= p
        else:
            out.append(enc_s(rng.randrange(P) & ~1))  # canonical and even: the square-root test decides
    return out


# ---- the model ------------------------------------------------------------------------------------------------------------
def test_model_multiples_of_g():
    """the reference's test_vectors_lib_decaf: its twisted chain G, G + G, .., and the untwisted encode([k]G0) and
    encode([-2k]B) give the 16 records; [2k]B does not (the sign convention the vectors decide)"""
    g = D.tw_decompress(GEN)
    acc = D.TW_IDENTITY
    for k, want in enumerate(MULTS):
        assert D.tw_compress(acc) == want, k
        assert D.tw_decompress(want) is not None and D.decode(want) is not None
        assert D.encode(M.mul(k, D.G0)) == want, k
        assert D.mul_gen(enc_s(k)) == want, k
        assert D.encode(D.decode(want)) == want
        acc = D.tw_add(acc, g)
    assert GEN == D.GENERATOR_BYTES == MULTS[1]
    assert [D.encode(M.mul(2 * k % L, M.B)) for k in range(1, 16)] != MULTS[1:]
    assert D.encode(M.mul(2, M.B)) != MULTS[1]


def test_model_invalid_points():
    for h in GOLDEN["invalid"]:
        assert D.tw_decompress(bytes.fromhex(h)) is None and D.decode(bytes.fromhex(h)) is None


def test_model_decoders_agree():
    """the twisted decompress and the untwisted decode give the same verdicts on 4,000 random records, the edge values,
    odd s and s >= p; every accepted record re-encodes to itself, through both representations"""
    recs = random_records(4000, 448) + edge_records()
    acc = 0
    for r in recs:
        t, u = D.tw_decompress(r), D.decode(r)
        assert (t is None) == (u is None), r.hex()
        if u is not None:
            acc += 1
            assert D.encode(u) == r and D.tw_compress(t) == r
    assert acc > 900
    assert D.decode(enc_s(1)) is None and D.decode(enc_s(P + 1)) is None and D.decode(enc_s(P - 1 + P % 2)) is None


def test_model_two_torsion_only():
    """[ell] decode(b) is (0, 1) or (0, -1); encode is invariant under adding (0, -1) but not (+-1, 0)"""
    rng = random.Random(2)
    seen = set()
    for r in [rand_point(rng) for _ in range(6)] + MULTS[1:6]:
        pt = D.decode(r)
        t = M.mul(L, pt)
        assert t in (M.IDENTITY, (0, P - 1))
        seen.add(t)
        assert D.encode(M.add(pt, (0, P - 1))) == r
        assert D.encode(M.add(pt, (1, 0))) != r
    assert len(seen) == 2


def test_model_generator_is_minus_two_b():
    assert D.encode(M.mul(L - 2, M.B)) == GEN
    assert M.add(M.mul(L - 2, M.B), M.neg(D.G0)) in (M.IDENTITY, (0, P - 1))


def test_model_scalar_acceptance():
    ok = [L - 1, 0, 1, 2**440]
    bad = [L, L + 1, 2**446, 2**448 - 1]
    for v in ok:
        assert D.scalar_ok(enc_s(v))
    for v in bad:
        assert not D.scalar_ok(enc_s(v))
    for top in (0x40, 0x80, 0xC0):
        r = bytearray(enc_s(5))
        r[55] |= top
        assert not D.scalar_ok(bytes(r))


def test_model_from_uniform_bytes():
    """the reference's seven RFC 9496 "group elements from uniform byte strings" vectors (DecafPoint::from_uniform_bytes)"""
    vecs = GOLDEN["from_uniform_bytes"]
    assert len(vecs) == 7
    for v in vecs:
        assert D.from_uniform_bytes(bytes.fromhex(v["input"])).hex() == v["output"]


def test_model_hash_vectors():
    """scalar_hash, the three DeriveKeyPair vectors replayed as the reference does (seed || I2OSP(len(info), 2) || info ||
    counter, the first nonzero scalar) and test_hash_to_curve's property"""
    sh = GOLDEN["scalar_hash"]
    assert D.hash_to_scalar(bytes.fromhex(sh["msg"]), bytes.fromhex(sh["dst"])).hex() == sh["scalar"]
    dk = GOLDEN["derive_key_pair"]
    seed, info = bytes.fromhex(dk["seed"]), bytes.fromhex(dk["info"])
    for v in dk["vectors"]:
        for c in range(256):
            s = D.hash_to_scalar(seed + len(info).to_bytes(2, "big") + info + bytes([c]), bytes.fromhex(v["dst"]))
            if int.from_bytes(s, "little"):
                break
        assert s.hex() == v["sk"]
    h = D.hash_to_curve(b"Hello, world!", b"test_hash_to_curve")
    assert h != ID and h != GEN and D.tw_decompress(h) is not None
    with pytest.raises(ValueError):
        D.hash_to_curve(b"x", b"")


# ---- device library and its host twin ---------------------------------------------------------------------------------------
class DecafDev:
    def __init__(self, kind):
        import __graft_entry__ as ge

        ge.build()
        self.kind = kind
        L_ = self.lib = ctypes.CDLL(os.path.join(DEV, "libecgdecaf448dev.so" if kind == "device" else "libecgdecaf448devsim.so"))
        sz = ctypes.c_size_t
        L_.dev_decaf_decode.argtypes = [sz, U8P, U32P, U8P]
        L_.dev_decaf_check.argtypes = [sz, U8P, U8P]
        L_.dev_decaf_encode.argtypes = [sz, U32P, U8P]
        L_.dev_decaf_mul.argtypes = [sz, U8P, U8P, ctypes.c_int, U32P, U32P]
        L_.dev_decaf_mul_xy.argtypes = [sz, U8P, U32P, U32P]
        L_.dev_decaf_fixed.argtypes = [sz, U8P, U32P, U32P, U32P]
        L_.dev_decaf_gen_scalar.argtypes = [sz, U8P, U8P]
        L_.dev_decaf_mod_l_64.argtypes = [sz, U8P, U8P]
        L_.dev_decaf_map.argtypes = [sz, U8P, U32P]
        L_.dev_decaf_xof.argtypes = [sz, U8P, U64P, U8P, ctypes.c_uint32, ctypes.c_int, U8P]
        L_.dev_decaf_hash.argtypes = [sz, U8P, U64P, U8P, ctypes.c_uint32, ctypes.c_int, U8P]
        L_.dev_decaf_from_uniform.argtypes = [sz, U8P, U8P]
        L_.dev_decaf_constants.argtypes = [U32P]
        L_.dev_decaf_error_string.restype = ctypes.c_char_p
        assert L_.dev_decaf_is_device() == (1 if kind == "device" else 0)

    def ok(self, rc):
        assert rc == 0, f"rc {rc}: {self.lib.dev_decaf_error_string(rc).decode()}"

    def constants(self):
        c = np.zeros(70, np.uint32)
        self.lib.dev_decaf_constants(_p(c, U32P))
        return [int.from_bytes(c[14 * i:14 * i + 14].tobytes(), "little") for i in range(5)]

    def decode(self, recs):
        xy, ok = np.zeros(28 * len(recs), np.uint32), np.zeros(len(recs), np.uint8)
        self.ok(self.lib.dev_decaf_decode(len(recs), _p(_arr(recs), U8P), _p(xy, U32P), _p(ok, U8P)))
        return [int(v) for v in ok], xy

    def check(self, recs):
        ok = np.zeros(len(recs), np.uint8)
        self.ok(self.lib.dev_decaf_check(len(recs), _p(_arr(recs), U8P), _p(ok, U8P)))
        return [int(v) for v in ok]

    def encode(self, soa, n):
        out = np.zeros(56 * n, np.uint8)
        self.ok(self.lib.dev_decaf_encode(n, _p(soa, U32P), _p(out, U8P)))
        return _rows(out)

    def mul(self, ks, ps, ct=False):
        n = len(ks)
        p = _arr(ps) if ps is not None else None
        ext, st = np.zeros(56 * n, np.uint32), np.zeros(2, np.uint32)
        self.ok(self.lib.dev_decaf_mul(n, _p(_arr(ks), U8P), _p(p, U8P) if p is not None else None, int(ct), _p(ext, U32P), _p(st, U32P)))
        return ext, [int(st[0]), int(st[1])]

    def mul_xy(self, ks, pts):
        n = len(ks)
        xy = np.frombuffer(b"".join(x.to_bytes(56, "little") + y.to_bytes(56, "little") for x, y in pts), np.uint32).copy()
        ext = np.zeros(56 * n, np.uint32)
        self.ok(self.lib.dev_decaf_mul_xy(n, _p(_arr(ks), U8P), _p(xy, U32P), _p(ext, U32P)))
        return ext

    def fixed(self, ks, table):
        n = len(ks)
        ext, st = np.zeros(56 * n, np.uint32), np.zeros(2, np.uint32)
        self.ok(self.lib.dev_decaf_fixed(n, _p(_arr(ks), U8P), _p(table, U32P), _p(ext, U32P), _p(st, U32P)))
        return ext, [int(st[0]), int(st[1])]

    def gen_scalar(self, ks):
        out = np.zeros(56 * len(ks), np.uint8)
        self.ok(self.lib.dev_decaf_gen_scalar(len(ks), _p(_arr(ks), U8P), _p(out, U8P)))
        return [int.from_bytes(r, "little") for r in _rows(out)]

    def mod_l_64(self, hs):
        out = np.zeros(56 * len(hs), np.uint8)
        self.ok(self.lib.dev_decaf_mod_l_64(len(hs), _p(_arr(hs), U8P), _p(out, U8P)))
        return [int.from_bytes(r, "little") for r in _rows(out)]

    def map(self, us):
        n = len(us)
        ext = np.zeros(56 * n, np.uint32)
        self.ok(self.lib.dev_decaf_map(n, _p(_arr(us), U8P), _p(ext, U32P)))
        return ext_points(ext, n)

    def _msgs(self, msgs):
        offs = np.zeros(len(msgs) + 1, np.uint64)
        offs[1:] = np.cumsum([len(m) for m in msgs])
        data = np.frombuffer(b"".join(msgs) + b"\0", np.uint8).copy()
        return data, offs

    def xof(self, msgs, suffix, length):
        data, offs = self._msgs(msgs)
        sfx = np.frombuffer(suffix, np.uint8).copy()
        out = np.zeros(288 * len(msgs), np.uint8)
        self.ok(self.lib.dev_decaf_xof(len(msgs), _p(data, U8P), _p(offs, U64P), _p(sfx, U8P), len(suffix), length, _p(out, U8P)))
        return [bytes(r[:length]) for r in out.reshape(-1, 288)]

    def from_uniform(self, us):
        out = np.zeros(56 * len(us), np.uint8)
        self.ok(self.lib.dev_decaf_from_uniform(len(us), _p(_arr(us), U8P), _p(out, U8P)))
        return _rows(out)

    def hash(self, msgs, suffix, mode):
        data, offs = self._msgs(msgs)
        sfx = np.frombuffer(suffix, np.uint8).copy()
        out = np.zeros(56 * len(msgs), np.uint8)
        self.ok(self.lib.dev_decaf_hash(len(msgs), _p(data, U8P), _p(offs, U64P), _p(sfx, U8P), len(suffix), mode, _p(out, U8P)))
        return _rows(out)


def _p(a, t):
    return a.ctypes.data_as(t)


def _arr(recs):
    return np.frombuffer(b"".join(recs), np.uint8).copy()


def _rows(a):
    return [bytes(r) for r in np.asarray(a, np.uint8).reshape(-1, 56)]


def ext_points(ext, n):
    w = np.asarray(ext, np.uint32).reshape(56, n)
    return [[int.from_bytes(w[14 * c:14 * c + 14, i].tobytes(), "little") for c in range(4)] for i in range(n)]


def to_soa(pts):
    n = len(pts)
    w = np.zeros((56, n), np.uint32)
    for i, p in enumerate(pts):
        for c in range(4):
            w[14 * c:14 * c + 14, i] = np.frombuffer((p[c] % P).to_bytes(56, "little"), np.uint32)
    return w.reshape(-1).copy()


def affine(e):
    X, Y, Z, T = e
    assert T * Z % P == X * Y % P
    zi = M.inv(Z)
    return X * zi % P, Y * zi % P


def proj_encode(e):
    return D.encode_ext(e[0], e[2], e[3])


_BACKENDS = {}


def backend(kind):
    if kind not in _BACKENDS:
        _BACKENDS[kind] = DecafDev(kind)
    return _BACKENDS[kind]


@pytest.fixture(scope="module", params=[pytest.param("host", id="host"), pytest.param("device", id="device", marks=pytest.mark.gpu)])
def be(request):
    return backend(request.param)


def test_dev_constants(be):
    assert be.constants() == [D.SQRT_MINUS_D, D.INV_SQRT_MINUS_D, D.DECAF_FACTOR, D.G0[0], D.G0[1]]


def test_dev_decode_and_check(be):
    recs = random_records(600, 9) + edge_records()
    ok, xy = be.decode(recs)
    assert be.check(recs) == ok
    w = xy.reshape(-1, 28)
    for i, r in enumerate(recs):
        want = D.decode(r)
        assert ok[i] == (want is not None), r.hex()
        if want is not None:
            got = (int.from_bytes(w[i, :14].tobytes(), "little"), int.from_bytes(w[i, 14:].tobytes(), "little"))
            assert got == want, r.hex()
    if be.kind == "device":
        assert np.array_equal(xy, backend("host").decode(recs)[1])


def test_dev_encode(be):
    """projective representatives with random Z, shifted by (0, -1) or not, and the identity in both 2-torsion forms"""
    rng = random.Random(3)
    pts = [D.decode(r) for r in MULTS] + [D.decode(rand_point(rng)) for _ in range(40)]
    pts += [M.add(p, (0, P - 1)) for p in pts[:20]] + [(0, P - 1)]
    exts = []
    for x, y in pts:
        z = rng.randrange(1, P)
        exts.append([x * z, y * z, z, x * y * z])
    got = be.encode(to_soa(exts), len(exts))
    assert got == [D.encode(p) for p in pts]
    assert got[:16] == MULTS and got[0] == ID and got[-1] == ID


def edge_scalars():
    ks = [0, 1, 2, 3, 4, L - 1, L - 2, L - 3, (L - 1) // 2, (L + 1) // 2, 2**445, 2**446 - 2**300]
    rng = random.Random(56)
    ks += [rng.randrange(L) for _ in range(12)]
    ks += [k ^ 1 for k in ks if k ^ 1 < L]
    return ks


def test_dev_mul_var(be):
    """ed448_mul_var on decoded points and on representatives shifted by (0, -1) at edge scalars of both parities, and the
    Decaf mul kernel (both paths) on the same pairs and on G0 (P56 = NULL)"""
    rng = random.Random(5)
    ks = edge_scalars()
    recs = [rand_point(rng) for _ in range(5)] + [ID, GEN]
    pairs = [(k, recs[i % len(recs)]) for i, k in enumerate(ks)]
    pts = [D.decode(r) for _, r in pairs]
    want = [D.encode(M.mul(k, pt)) for (k, _), pt in zip(pairs, pts)]
    k56 = [enc_s(k) for k, _ in pairs]
    ext = be.mul_xy(k56, pts)
    assert [proj_encode(e) for e in ext_points(ext, len(pairs))] == want
    shifted = [M.add(pt, (0, P - 1)) for pt in pts]
    ext2 = be.mul_xy(k56, shifted)
    assert [proj_encode(e) for e in ext_points(ext2, len(pairs))] == want
    extk, st = be.mul(k56, [r for _, r in pairs])
    assert st == [0, 0xFFFFFFFF]
    assert be.encode(extk, len(pairs)) == want
    extc, _ = be.mul(k56, [r for _, r in pairs], ct=True)
    assert be.encode(extc, len(pairs)) == want
    extg, _ = be.mul(k56[:24], None)
    assert be.encode(extg, 24) == [D.mul_gen(enc_s(k)) for k in ks[:24]]
    if be.kind == "device":
        assert np.array_equal(extk, backend("host").mul(k56, [r for _, r in pairs])[0])


def test_dev_mul_reports_refusals(be):
    ks = [enc_s(3)] * 8
    ps = [GEN] * 8
    ks[5] = enc_s(L)
    ps[6] = enc_s(1)
    assert be.mul(ks, ps)[1] == [3, 5]
    ks[5] = enc_s(1)
    assert be.mul(ks, ps)[1] == [2, 6]
    ps[2] = enc_s(P + 1)
    assert be.mul(ks, ps)[1] == [2, 2]


@pytest.fixture(scope="module")
def model_table():
    return np.frombuffer(G.fixed_base_table(8, 56), np.uint32).copy()


def test_dev_fixed_base_and_transform(be, model_table):
    """the scalar transform k -> (-2k) mod ell and the fixed-base kernel over a model-built Ed448 table"""
    ks = edge_scalars() + list(range(16))
    assert be.gen_scalar([enc_s(k) for k in ks]) == [D.gen_scalar(k) for k in ks]
    ext, st = be.fixed([enc_s(k) for k in ks], model_table)
    assert st == [0, 0xFFFFFFFF]
    got = be.encode(ext, len(ks))
    assert got == [D.mul_gen(enc_s(k)) for k in ks]
    assert got[-16:] == MULTS
    assert be.fixed([enc_s(1), enc_s(L + 5), enc_s(2**447)], model_table)[1] == [1, 1]


def test_dev_map(be):
    rng = random.Random(7)
    us = [0, 1, 2, P - 1, P, P + 1, 2**448 - 1] + [rng.getrandbits(448) for _ in range(60)]
    got = be.map([enc_s(u) for u in us])
    for u, e in zip(us, got):
        want = D.tw_map(u)
        assert D.tw_on_curve(tuple(v % P for v in e))
        assert D.tw_compress(e) == D.tw_compress(want)
        assert [v % P for v in e] == list(want), u


def test_dev_expand_message_xof(be):
    """message lengths around the SHAKE256 rate (136), DST lengths 1, 255 and 256 (oversize: the hashed DST' in the
    suffix), every output length the entries use, and outputs past one block: 168 (the edwards448 RO suite's 2 x 84) and
    280 (past two), each against hashlib's SHAKE256 over the message and the suffix"""
    import hashlib

    rng = random.Random(8)
    msgs = [bytes(rng.getrandbits(8) for _ in range(n)) for n in (0, 135, 136, 137, 271, 272, 273)]
    for dst in (b"D", bytes(range(255)), bytes(256)):
        for length in (56, 64, 112, 168, 280):
            sfx = D.xof_suffix(dst, length)
            got = be.xof(msgs, sfx, length)
            assert got == [D.expand_message_xof(m, dst, length) for m in msgs], (len(dst), length)
            assert got == [hashlib.shake_256(m + sfx).digest(length) for m in msgs], (len(dst), length)


def test_dev_from_uniform_bytes(be):
    """the RO path after expansion (two maps, one twisted addition, compress) on the reference's seven RFC 9496
    uniform-bytes vectors, and random strings against the model"""
    vecs = GOLDEN["from_uniform_bytes"]
    assert be.from_uniform([bytes.fromhex(v["input"]) for v in vecs]) == [bytes.fromhex(v["output"]) for v in vecs]
    rng = random.Random(112)
    us = [rng.getrandbits(896).to_bytes(112, "little") for _ in range(40)] + [b"\xff" * 112, bytes(112)]
    assert be.from_uniform(us) == [D.from_uniform_bytes(u) for u in us]


def test_dev_mod_l_64(be):
    hs = [b"\xff" * 64, bytes(64)]
    for e in range(0, 67):
        for d in (-1, 0, 1):
            v = L * (1 << e) + d
            if 0 <= v < 2**512:
                hs.append(v.to_bytes(64, "little"))
    rng = random.Random(64)
    hs += [rng.getrandbits(512).to_bytes(64, "little") for _ in range(100)]
    assert be.mod_l_64(hs) == [int.from_bytes(h, "little") % L for h in hs]


def test_dev_hash_kernels(be):
    rng = random.Random(12)
    msgs = [bytes(rng.getrandbits(8) for _ in range(n)) for n in (0, 1, 13, 135, 136, 137, 300)]
    msgs.append(b"Hello, world!")
    for dst in (RO, b"test_hash_to_curve", bytes(300)):
        assert be.hash(msgs, D.xof_suffix(dst, 112), 0) == [D.hash_to_curve(m, dst) for m in msgs]
        assert be.hash(msgs, D.xof_suffix(dst, 56), 1) == [D.hash_to_curve(m, dst, True) for m in msgs]
        assert be.hash(msgs, D.xof_suffix(dst, 64), 2) == [D.hash_to_scalar(m, dst) for m in msgs]
    if be.kind == "device":
        h = backend("host")
        assert be.hash(msgs, D.xof_suffix(RO, 112), 0) == h.hash(msgs, D.xof_suffix(RO, 112), 0)


# ---- the C ABI, the Python and C++ mirrors ----------------------------------------------------------------------------------
def test_abi_null_ctx():
    import ecgpu

    lib = ecgpu.load_library()
    z = np.zeros(128, np.uint8)
    o = np.zeros(2, np.uint64)
    d = z.ctypes.data
    assert lib.ecg_decaf448_mul_batch(None, 1, d, d, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_decaf448_mul_gen_batch(None, 1, d, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_decaf448_lincomb(None, 1, d, d, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_decaf448_check_batch(None, 1, d, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_decaf448_hash_to_curve_batch(None, 1, d, o.ctypes.data, d, 1, 0, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_decaf448_hash_to_scalar_batch(None, 1, d, o.ctypes.data, d, 1, d) == ecgpu.ECG_EINVAL


CPP = r"""
#include "ecgpu.hpp"
#include <cstdio>
int main() {
  try {
    ecgpu::Engine eng(ECG_SECP256K1);
    using B = ecgpu::Engine::Decaf448Bytes;
    std::vector<B> k(3);
    k[0][0] = 1;
    k[1][0] = 2;
    auto g = eng.decaf448_mul_gen(k);
    std::vector<B> P = {g[0], g[0], g[1]};
    auto m = eng.decaf448_mul(k, P);
    auto s = eng.decaf448_lincomb(k, P);
    auto e = eng.decaf448_lincomb({}, {});
    B bad{};
    bad[0] = 1;
    auto ok = eng.decaf448_check({g[0], bad, e});
    std::vector<uint8_t> msg = {'h', 'e', 'l', 'l', 'o', ' ', 'w', 'o', 'r', 'l', 'd'};
    std::string d = "decaf448_XOF:SHAKE256_D448MAP_RO_";
    auto hs = eng.decaf448_hash_to_scalar({msg}, std::vector<uint8_t>(d.begin(), d.end()));
    auto hc = eng.decaf448_hash_to_curve({msg, {}}, std::vector<uint8_t>(d.begin(), d.end()));
    std::printf("gen=%%d mul=%%d lin=%%d id=%%d chk=%%d h2s=%%02x%%02x h2c=%%d\n", (int)(g[0][0] == 0x66 && g[2][0] == 0),
                (int)(m[1] == g[1] && m[2][0] == 0), (int)(s == eng.decaf448_mul_gen({B{3}})[0]), (int)(e == B{}),
                (int)(ok[0] && !ok[1] && ok[2]), hs[0][0], hs[0][1], (int)(eng.decaf448_check(hc)[0] && eng.decaf448_check(hc)[1]));
    return 0;
  } catch (const ecgpu::Error& e) {
    std::printf("error %%d\n", (int)e.code);
    return e.code == ECG_ECUDA ? 42 : 3;  // 42: no GPU -> a loud failure, no CPU fallback
  }
}
"""


def _cpp_run():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "g.cpp"), os.path.join(d, "g")
        open(src, "w").write(CPP % {})
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "elliptic-curves_b200", "host"), src, LIB,
                               "-Wl,-rpath," + os.path.dirname(LIB), "-o", exe])
        p = subprocess.run([exe], capture_output=True, text=True, timeout=300)
        return p.returncode, p.stdout + p.stderr


def test_cpp_mirror_decaf448_compiles_and_links():
    import torch

    rc, out = _cpp_run()
    if torch.cuda.is_available():
        assert rc == 0, out
    else:
        assert rc == 42, out  # ECG_ECUDA without a GPU


@pytest.mark.gpu
def test_cpp_mirror_decaf448_for_real():
    rc, out = _cpp_run()
    assert rc == 0, out
    assert "gen=1 mul=1 lin=1 id=1 chk=1 h2s=55e7 h2c=1" in out


@pytest.fixture(scope="module")
def eng():
    import ecgpu

    e = ecgpu.Engine([0])
    yield e
    e.close()


def recs(ks):
    return _arr([enc_s(k) for k in ks])


@pytest.mark.gpu
def test_abi_fixtures(eng):
    assert _rows(eng.decaf448_mul_gen(recs(range(16)))) == MULTS
    assert _rows(eng.decaf448_mul(recs(range(16)), _arr([GEN] * 16))) == MULTS
    assert _rows(eng.decaf448_mul(recs([1] * 16), _arr(MULTS))) == MULTS
    assert list(eng.decaf448_check(_arr(MULTS + [bytes.fromhex(h) for h in GOLDEN["invalid"]]))) == [1] * 16 + [0, 0]
    sh = GOLDEN["scalar_hash"]
    assert bytes(eng.decaf448_hash_to_scalar([bytes.fromhex(sh["msg"])], bytes.fromhex(sh["dst"]))[0]).hex() == sh["scalar"]
    dk = GOLDEN["derive_key_pair"]
    seed, info = bytes.fromhex(dk["seed"]), bytes.fromhex(dk["info"])
    msgs = [seed + len(info).to_bytes(2, "big") + info + bytes([c]) for c in range(256)]
    for v in dk["vectors"]:
        out = _rows(eng.decaf448_hash_to_scalar(msgs, bytes.fromhex(v["dst"])))
        first = next(r for r in out if any(r))
        assert first.hex() == v["sk"]
    h = bytes(eng.decaf448_hash_to_curve([b"Hello, world!"], b"test_hash_to_curve")[0])
    assert h == D.hash_to_curve(b"Hello, world!", b"test_hash_to_curve") and h != ID and h != GEN


@pytest.fixture(scope="module")
def keyset(eng):
    """2^16 secret scalars a and their public elements [a]G from the device (checked against the model on a sample)"""
    rng = random.Random(65536)
    a = [rng.randrange(L) for _ in range(1 << 16)]
    a[:4] = [0, 1, 2, L - 1]
    pubs = _rows(eng.decaf448_mul_gen(recs(a)))
    return a, pubs


@pytest.mark.gpu
def test_abi_mul_gen_against_ed448(eng, keyset):
    """[k]G on 2^16 random k: the variable-base path on G gives the same bytes, and so does the model's encode of the
    Ed448 entry's [(-2k) mod ell]B"""
    a, pubs = keyset
    assert _rows(eng.decaf448_mul(recs(a), _arr([GEN] * len(a)))) == pubs
    ed = eng.ed448_mul_gen(_arr([G.enc_scalar(D.gen_scalar(k)) for k in a]))
    for i in range(len(a)):
        pt = M.decompress_unchecked(bytes(ed[i]))
        assert D.encode(pt) == pubs[i], i
    assert [D.mul_gen(enc_s(k)) for k in a[:64]] == pubs[:64]


@pytest.mark.gpu
def test_abi_mul_identity(eng, keyset):
    """[k]([a]G) == [k a mod ell]G over 2^16 pairs, and 256 against the model"""
    a, pubs = keyset
    rng = random.Random(7)
    ks = [rng.randrange(L) for _ in a]
    ks[:6] = [0, 1, 2, L - 1, L - 2, 4]
    got = _rows(eng.decaf448_mul(recs(ks), _arr(pubs)))
    want = _rows(eng.decaf448_mul_gen(recs([k * ai % L for k, ai in zip(ks, a)])))
    assert got == want
    for i in range(256):
        assert got[i] == D.mul(enc_s(ks[i]), pubs[i]), i


@pytest.mark.gpu
def test_abi_lincomb(eng, keyset):
    """n = 0, 1, 2, 57, 1,000 and 2^16 against mul_gen(sum k_i a_i); small n against the model as well"""
    a, pubs = keyset
    assert bytes(eng.decaf448_lincomb(np.zeros(0, np.uint8), np.zeros(0, np.uint8))) == ID
    rng = random.Random(57)
    for n in (1, 2, 57, 1000, 1 << 16):
        idx = [rng.randrange(len(a)) for _ in range(n)]
        ks = [rng.randrange(L) if i % 5 else [0, 1, L - 1, 2, 3][i // 5 % 5] for i in range(n)]
        got = bytes(eng.decaf448_lincomb(recs(ks), _arr([pubs[j] for j in idx])))
        s = sum(k * a[j] for k, j in zip(ks, idx)) % L
        assert got == bytes(eng.decaf448_mul_gen(recs([s]))[0]), n
        if n <= 57:
            assert got == D.lincomb([enc_s(k) for k in ks], [pubs[j] for j in idx])
    assert bytes(eng.decaf448_lincomb(recs([3, L - 3]), _arr([GEN, GEN]))) == ID


@pytest.mark.gpu
def test_abi_check_batch(eng):
    rs = random_records(1 << 16, 16) + edge_records()
    got = list(eng.decaf448_check(_arr(rs)))
    want = [int(D.decode(r) is not None) for r in rs]
    assert got == want
    assert sum(want) > 10000


@pytest.mark.gpu
def test_abi_hash(eng):
    """RO, NU and hash to scalar on 4,096 messages of mixed lengths against the model, under a short, a 255-byte and an
    oversize DST"""
    rng = random.Random(4096)
    lens = [0, 1, 135, 136, 137, 272, 1000] + [rng.randrange(0, 300) for _ in range(4089)]
    msgs = [bytes(rng.getrandbits(8) for _ in range(n)) for n in lens]
    for dst in (RO, bytes(range(255)), bytes(range(256)) * 2):
        sample = range(0, 4096, 1 if dst == RO else 16)
        ro = _rows(eng.decaf448_hash_to_curve(msgs, dst))
        nu = _rows(eng.decaf448_hash_to_curve(msgs, dst, nonuniform=True))
        sc = _rows(eng.decaf448_hash_to_scalar(msgs, dst))
        for i in sample:
            assert ro[i] == D.hash_to_curve(msgs[i], dst), i
            assert nu[i] == D.hash_to_curve(msgs[i], dst, True), i
            assert sc[i] == D.hash_to_scalar(msgs[i], dst), i
        assert all(eng.decaf448_check(_arr(ro[:256])))


@pytest.mark.gpu
def test_abi_rejected_inputs(eng):
    import ecgpu

    n = 300
    k = recs([5] * n)
    P_ = _arr([GEN] * n)
    bad_k = [enc_s(L), bytes(55) + b"\x40", bytes(55) + b"\xc0"]
    bad_p = [enc_s(1), enc_s(P + 1), enc_s(P - 1 + 1), bytes.fromhex(GOLDEN["invalid"][0]), bytes.fromhex(GOLDEN["invalid"][1])]
    cases = [(10 + i, "k", r) for i, r in enumerate(bad_k)] + [(20 + i, "P", r) for i, r in enumerate(bad_p)]
    for idx, what, rec in cases:
        for first in (idx, 250):
            kk, pp = k.copy(), P_.copy()
            for j in (first, 299):
                (kk if what == "k" else pp)[56 * j:56 * j + 56] = np.frombuffer(rec, np.uint8)
            err = ecgpu.ScalarRangeError if what == "k" else ecgpu.NotOnCurveError
            with pytest.raises(err) as ei:
                eng.decaf448_mul(kk, pp)
            assert ei.value.index == first
            if what == "k":
                with pytest.raises(err) as ei:
                    eng.decaf448_mul_gen(kk)
                assert ei.value.index == first
            with pytest.raises(err) as ei:
                eng.decaf448_lincomb(kk, pp)
            assert ei.value.index == first
    assert _rows(eng.decaf448_mul(k[:56], P_[:56]))[0] == MULTS[5]  # the engine still works


def _wave(minblk):
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count * minblk * 128


@pytest.mark.gpu
def test_abi_ragged_sizes(eng):
    """sizes across the host chunks (a wave is sm_count * 2 * 128 elements), n = 0"""
    n0 = _wave(2)
    rng = random.Random(n0)
    base = [rand_point(rng) for _ in range(8)]
    for n in (0, 1, 129, 2 * n0 + 5, 4 * n0 + 3):
        ks = [rng.randrange(L) for _ in range(n)]
        pts = [base[i % 8] for i in range(n)]
        out = _rows(eng.decaf448_mul(recs(ks), _arr(pts)))
        gen = _rows(eng.decaf448_mul_gen(recs(ks)))
        chk = eng.decaf448_check(_arr(pts))
        assert len(out) == len(gen) == len(chk) == n
        for i in list(range(0, n, max(1, n // 40))) + ([n - 1] if n else []):
            assert out[i] == D.mul(enc_s(ks[i]), pts[i]), (n, i)
            assert gen[i] == D.mul_gen(enc_s(ks[i])), (n, i)
        assert all(chk)
        msgs = [bytes([i & 0xFF]) * (i % 7) for i in range(n)]
        h = _rows(eng.decaf448_hash_to_curve(msgs, RO))
        for i in list(range(0, n, max(1, n // 20))) + ([n - 1] if n else []):
            assert h[i] == D.hash_to_curve(msgs[i], RO), (n, i)


@pytest.mark.gpu
def test_abi_device_pointers():
    import torch

    import ecgpu

    rng = random.Random(99)
    n = 4099
    ks = [rng.randrange(L) for _ in range(n)]
    pts = [rand_point(rng) for _ in range(16)]
    pts = [pts[i % 16] for i in range(n)]
    msgs = [bytes([i & 0xFF]) * (i % 150) for i in range(n)]
    h = ecgpu.Engine([0])
    want = (h.decaf448_mul(recs(ks), _arr(pts)), h.decaf448_mul_gen(recs(ks)), h.decaf448_lincomb(recs(ks), _arr(pts)),
            h.decaf448_hash_to_curve(msgs, RO), h.decaf448_hash_to_curve(msgs, RO, True), h.decaf448_hash_to_scalar(msgs, RO))
    h.close()
    e = ecgpu.Engine([0], device_ptrs=True)
    # 56-byte records in device memory are 4-byte aligned (as X448's); misaligned ones are ECG_EINVAL
    kd = torch.zeros(56 * n + 4, dtype=torch.uint8, device="cuda")
    kd[4:] = torch.from_numpy(recs(ks)).cuda()
    pd = torch.zeros(56 * n + 8, dtype=torch.uint8, device="cuda")
    pd[8:] = torch.from_numpy(_arr(pts)).cuda()
    od = torch.zeros(56 * n + 4, dtype=torch.uint8, device="cuda")
    launches = e.kernel_launches
    e.decaf448_mul_ptr(n, kd.data_ptr() + 4, pd.data_ptr() + 8, od.data_ptr() + 4)
    torch.cuda.synchronize()
    assert e.kernel_launches == launches + 2  # the scalar multiplication and the encoding
    assert np.array_equal(od[4:].cpu().numpy(), want[0].reshape(-1))
    e.decaf448_mul_gen_ptr(n, kd.data_ptr() + 4, od.data_ptr() + 4)
    torch.cuda.synchronize()
    assert np.array_equal(od[4:].cpu().numpy(), want[1].reshape(-1))
    o1 = torch.zeros(60, dtype=torch.uint8, device="cuda")
    e.decaf448_lincomb_ptr(n, kd.data_ptr() + 4, pd.data_ptr() + 8, o1.data_ptr() + 4)
    torch.cuda.synchronize()
    assert np.array_equal(o1[4:].cpu().numpy(), want[2])
    o1.fill_(7)
    e.decaf448_lincomb_ptr(0, 0, 0, o1.data_ptr() + 4)
    torch.cuda.synchronize()
    assert bytes(o1[4:].cpu().numpy()) == ID
    okd = torch.zeros(n, dtype=torch.uint8, device="cuda")
    e.decaf448_check_ptr(n, pd.data_ptr() + 8, okd.data_ptr())
    torch.cuda.synchronize()
    assert okd.cpu().numpy().all()
    data, offs = ecgpu.Engine._pack_messages(msgs)
    dd = torch.from_numpy(data).cuda()
    do = torch.from_numpy(offs.view(np.int64)).cuda()
    for nu, w in ((False, want[3]), (True, want[4])):
        e.decaf448_hash_to_curve_ptr(n, dd.data_ptr(), do.data_ptr(), od.data_ptr() + 4, RO, nu)
        torch.cuda.synchronize()
        assert np.array_equal(od[4:].cpu().numpy(), w.reshape(-1))
    e.decaf448_hash_to_scalar_ptr(n, dd.data_ptr(), do.data_ptr(), od.data_ptr() + 4, RO)
    torch.cuda.synchronize()
    assert np.array_equal(od[4:].cpu().numpy(), want[5].reshape(-1))
    bad = kd.clone()
    bad[4 + 56 * 7:4 + 56 * 7 + 56] = 0xFF
    with pytest.raises(ecgpu.ScalarRangeError) as ei:
        e.decaf448_mul_ptr(n, bad.data_ptr() + 4, pd.data_ptr() + 8, od.data_ptr() + 4)
    assert ei.value.index == 7
    with pytest.raises(ecgpu.EcgError) as ei:
        e.decaf448_mul_ptr(n, kd.data_ptr() + 1, pd.data_ptr() + 8, od.data_ptr() + 4)
    assert ei.value.code == ecgpu.ECG_EINVAL
    e.close()


@pytest.mark.gpu
def test_abi_consttime_and_zeroize_identical(eng):
    import ecgpu

    rng = random.Random(2051)
    n = 2051
    ks = [rng.randrange(L) for _ in range(n)]
    ks[:4] = [0, 1, 2, L - 1]
    pts = [rand_point(rng) for _ in range(8)] + [ID]
    pts = [pts[i % 9] for i in range(n)]
    msgs = [bytes([i & 0xFF]) * (i % 40) for i in range(n)]

    def run(e):
        return (e.decaf448_mul(recs(ks), _arr(pts)), e.decaf448_mul_gen(recs(ks)), e.decaf448_lincomb(recs(ks), _arr(pts)),
                e.decaf448_check(_arr(pts)), e.decaf448_hash_to_curve(msgs, RO), e.decaf448_hash_to_scalar(msgs, RO))

    base = run(eng)
    for kw in ({"zeroize": True}, {"consttime": True}, {"zeroize": True, "consttime": True}):
        e = ecgpu.Engine([0], **kw)
        for g, b in zip(run(e), base):
            assert np.array_equal(g, b), kw
        e.close()


@pytest.mark.gpu
def test_abi_einval(eng):
    import ecgpu

    lib, c = eng.lib, eng._ctx
    z, ids = np.zeros(56 * 2, np.uint8), _arr([ID, ID])
    d = z.ctypes.data
    o = np.array([0, 1, 2], np.uint64)
    dst = np.frombuffer(RO, np.uint8).copy()
    assert lib.ecg_decaf448_mul_batch(c, 2, d, ids.ctypes.data, d) == ecgpu.ECG_OK
    for args in ((None, d, d), (d, None, d), (d, d, None)):
        assert lib.ecg_decaf448_mul_batch(c, 2, *args) == ecgpu.ECG_EINVAL
        assert lib.ecg_decaf448_lincomb(c, 2, *args) == ecgpu.ECG_EINVAL
    assert lib.ecg_decaf448_mul_gen_batch(c, 2, None, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_decaf448_mul_gen_batch(c, 2, d, None) == ecgpu.ECG_EINVAL
    assert lib.ecg_decaf448_check_batch(c, 2, None, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_decaf448_check_batch(c, 2, d, None) == ecgpu.ECG_EINVAL
    for n in (0, 2):
        assert lib.ecg_decaf448_hash_to_curve_batch(c, n, d, o.ctypes.data, dst.ctypes.data, 0, 0, d) == ecgpu.ECG_EINVAL  # EmptyDst
        assert lib.ecg_decaf448_hash_to_curve_batch(c, n, d, o.ctypes.data, None, 5, 0, d) == ecgpu.ECG_EINVAL
        assert lib.ecg_decaf448_hash_to_scalar_batch(c, n, d, o.ctypes.data, dst.ctypes.data, 0, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_decaf448_hash_to_curve_batch(c, 2, d, None, dst.ctypes.data, dst.size, 0, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_decaf448_hash_to_curve_batch(c, 2, d, o.ctypes.data, dst.ctypes.data, dst.size, 0, None) == ecgpu.ECG_EINVAL
    assert lib.ecg_decaf448_hash_to_scalar_batch(c, 2, None, o.ctypes.data, dst.ctypes.data, dst.size, d) == ecgpu.ECG_EINVAL  # null msgs
    dec = np.array([0, 2, 1], np.uint64)
    assert lib.ecg_decaf448_hash_to_scalar_batch(c, 2, d, dec.ctypes.data, dst.ctypes.data, dst.size, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_decaf448_mul_batch(c, 0, None, None, None) == ecgpu.ECG_OK
    assert lib.ecg_decaf448_mul_gen_batch(c, 0, None, None) == ecgpu.ECG_OK
    assert lib.ecg_decaf448_check_batch(c, 0, None, None) == ecgpu.ECG_OK
    assert lib.ecg_decaf448_hash_to_curve_batch(c, 0, None, None, dst.ctypes.data, dst.size, 0, None) == ecgpu.ECG_OK
    big = np.zeros(300, np.uint8)  # an oversize DST with nothing to hash launches nothing
    launches = eng.kernel_launches
    assert lib.ecg_decaf448_hash_to_curve_batch(c, 0, None, None, big.ctypes.data, big.size, 0, None) == ecgpu.ECG_OK
    assert lib.ecg_decaf448_hash_to_scalar_batch(c, 0, None, None, big.ctypes.data, big.size, None) == ecgpu.ECG_OK
    assert eng.kernel_launches == launches
    z[:56] = 9
    assert lib.ecg_decaf448_lincomb(c, 0, None, None, d) == ecgpu.ECG_OK
    assert lib.ecg_decaf448_lincomb(c, 0, None, None, None) == ecgpu.ECG_EINVAL
    assert bytes(z[:56]) == ID


@pytest.mark.gpu
def test_abi_multi_device():
    """two shards (two GPUs when present, else two contexts of device 0): byte-identical to one device, refusals with
    their index in the whole batch"""
    import torch

    import ecgpu

    devs = [0, 1] if torch.cuda.device_count() >= 2 else [0, 0]
    rng = random.Random(2)
    n = 5003
    ks = [rng.randrange(L) for _ in range(n)]
    pts = [rand_point(rng) for _ in range(8)]
    pts = [pts[i % 8] for i in range(n)]
    msgs = [bytes([i & 0xFF]) * (i % 33) for i in range(n)]
    one, two = ecgpu.Engine([0]), ecgpu.Engine(devs)
    for f in (lambda e: e.decaf448_mul(recs(ks), _arr(pts)), lambda e: e.decaf448_mul_gen(recs(ks)),
              lambda e: e.decaf448_lincomb(recs(ks), _arr(pts)), lambda e: e.decaf448_check(_arr(pts)),
              lambda e: e.decaf448_hash_to_curve(msgs, bytes(300)), lambda e: e.decaf448_hash_to_scalar(msgs, RO)):
        assert np.array_equal(f(one), f(two))
    bad = recs(ks)
    bad[56 * 4000:56 * 4001] = 0xFF
    with pytest.raises(ecgpu.ScalarRangeError) as ei:
        two.decaf448_mul(bad, _arr(pts))
    assert ei.value.index == 4000
    one.close()
    two.close()
