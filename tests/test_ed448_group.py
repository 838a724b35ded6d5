"""Ed448 group operations (EdwardsPoint): the model (ed448_group_model.py) against the reference's semantics, the device
kernels (tests/dev/ed448_group_dev.cu: decompression, the scalar check, the variable-base and fixed-base routines, the sum
and the normalisation, under the production launch bounds) against their host twin and the model, and
ecg_ed448_mul_batch / ecg_ed448_mul_gen_batch / ecg_ed448_lincomb through the C ABI, the Python and C++ mirrors.

Oracles: the RFC 8032 public keys of the reference's vectors (tests/golden/ed448.json), OpenSSL's Ed448 key generation
through `cryptography` (independent of this code), the model in Python integers, and algebraic identities between the
entries ([k]([s]B) == [k s]B, sum k_i [s_i]B == [sum k_i s_i]B)."""
import ctypes
import json
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

import ed448_group_model as G
import ed448_model as M

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = os.path.join(HERE, "dev")
LIB = os.path.join(ROOT, "elliptic-curves_b200", "libecgpu.so")
GOLDEN = json.load(open(os.path.join(HERE, "golden", "ed448.json")))
U8P = ctypes.POINTER(ctypes.c_uint8)
U32P = ctypes.POINTER(ctypes.c_uint32)
P, L = M.P, M.L
ID = G.IDENTITY_BYTES


def enc_y(y: int, sign: int = 0, low: int = 0) -> bytes:
    return y.to_bytes(56, "little") + bytes([(sign << 7) | low])


def openssl_public(seed: bytes) -> bytes:
    from cryptography.hazmat.primitives.asymmetric.ed448 import Ed448PrivateKey

    return Ed448PrivateKey.from_private_bytes(seed).public_key().public_bytes_raw()


def non_decodable_y():
    """the smallest y >= 2 with no x: (1 - y^2) / (1 - d y^2) is not a square"""
    y = 2
    while M.decompress_unchecked(enc_y(y)) is not None:
        y += 1
    return y


def rand_point(rng):
    return M.mul(rng.randrange(1, L), M.B)


def edge_scalars():
    """0, 1, 2, ell - 1, ell - 2, powers of two and window-boundary patterns (runs of ones and zeros across 4-bit and
    8-bit windows), and odd / even pairs around the add-ell step"""
    ks = [0, 1, 2, 3, 4, 15, 16, 17, L - 1, L - 2, L - 3, (L - 1) // 2, (L + 1) // 2, 2**445, 2**446 - 2**300, L - 2**200]
    ks += [2**i for i in (3, 4, 7, 8, 63, 64, 223, 224, 440, 444)]
    ks += [(2**i - 1) for i in (4, 8, 12, 100, 444)]
    ks += [int("f0" * 55, 16), int("0f" * 55, 16), int("8" + "0" * 110, 16) + 1, int("7" + "f" * 110, 16)]
    rng = random.Random(112)
    ks += [rng.randrange(L) for _ in range(16)]
    ks = [k % L for k in ks]
    ks += [k ^ 1 for k in ks if k ^ 1 < L]  # the other parity of every case
    return ks


# ---- the model ------------------------------------------------------------------------------------------------------------
def test_scalar_acceptance():
    """the reference's from_canonical_bytes and the simplified rule agree: byte 56 is ignored, bytes 0..55 must be < ell"""
    rng = random.Random(57)
    cases = [G.enc_scalar(v, b) for v in (0, 1, L - 1, L, L + 1, 2**446 - 1, 2**446, 2**448 - 1) for b in (0, 1, 0x80, 0xFF)]
    cases += [bytes(rng.getrandbits(8) for _ in range(57)) for _ in range(2000)]
    cases += [rng.getrandbits(446).to_bytes(56, "little") + bytes([rng.getrandbits(8)]) for _ in range(2000)]
    for c in cases:
        assert G.from_canonical_bytes(c) == G.scalar_ok(c), c.hex()
    assert G.scalar_ok(G.enc_scalar(L - 1)) and not G.scalar_ok(G.enc_scalar(L)) and not G.scalar_ok(G.enc_scalar(2**446))
    # byte 56 = 0xFF with a small scalar is accepted and gives the same output as byte 56 = 0
    assert G.scalar_ok(G.enc_scalar(5, 0xFF))
    assert G.mul_gen(G.enc_scalar(5, 0xFF)) == G.mul_gen(G.enc_scalar(5)) == M.encode(M.mul(5, M.B))


def test_point_acceptance():
    """the identity under both sign bits, (0, -1), the all-zero record, P + T for each torsion point T, y >= p and bits
    0-6 of byte 56"""
    assert G.decompress(ID) == M.IDENTITY
    assert G.decompress(enc_y(1, 1)) == M.IDENTITY
    assert G.decompress(enc_y(1, 1, 0x7F)) == M.IDENTITY
    assert G.decompress(enc_y(P - 1)) is None and G.decompress(enc_y(P - 1, 1)) is None  # (0, -1), order 2
    assert G.decompress(bytes(57)) is None  # CompressedEdwardsY::IDENTITY: y = 0, a point of order 4
    assert G.decompress(enc_y(P + 1)) == M.IDENTITY  # y >= p is reduced
    rng = random.Random(4)
    for _ in range(10):
        pt = rand_point(rng)
        e = M.encode(pt)
        assert G.decompress(e) == pt
        assert G.decompress(e[:56] + bytes([e[56] | 0x55])) == pt
        if pt[1] + P < 2**448:
            assert G.decompress(enc_y(pt[1] + P, e[56] >> 7)) == pt
        for T in M.TORSION:
            assert G.decompress(M.encode(M.add(pt, T))) is None


def test_isogeny_scalar_mul_is_plain_mul_on_the_subgroup():
    """[4 (s / 4 mod ell)]P == [s]P on subgroup points, and not on their torsion translates (why the decoder matters)"""
    rng = random.Random(1)
    for _ in range(6):
        pt = rand_point(rng)
        for s in (0, 1, 2, 3, L - 1, rng.randrange(L), rng.getrandbits(446)):
            assert G.reference_scalar_mul(s, pt) == M.mul(s, pt)
    q = M.add(rand_point(rng), M.TORSION[1])
    assert G.reference_scalar_mul(1, q) != M.mul(1, q)


def test_rfc_public_keys():
    """public = compress([clamp(SHAKE256(seed)[:57]) mod ell] B) for the RFC 8032 vectors of the reference"""
    for v in GOLDEN["vectors"]:
        a = G.secret_scalar(bytes.fromhex(v["seed"]))
        assert G.mul_gen(G.enc_scalar(a)).hex() == v["public"]


def test_openssl_keypairs():
    rng = random.Random(448)
    for _ in range(1024):
        seed = rng.getrandbits(456).to_bytes(57, "little")
        assert G.mul_gen(G.enc_scalar(G.secret_scalar(seed))) == openssl_public(seed)


# ---- device library and its host twin ---------------------------------------------------------------------------------------
class GroupDev:
    def __init__(self, kind):
        import __graft_entry__ as ge

        ge.build()
        self.kind = kind
        L_ = self.lib = ctypes.CDLL(os.path.join(DEV, "libecged448gdev.so" if kind == "device" else "libecged448gdevsim.so"))
        sz = ctypes.c_size_t
        L_.dev_ed448g_scalar_ok.argtypes = [sz, U8P, U8P]
        L_.dev_ed448g_decompress.argtypes = [sz, U8P, U32P, U8P]
        L_.dev_ed448g_mul.argtypes = [sz, U8P, U8P, ctypes.c_int, U32P, U32P]
        L_.dev_ed448g_fixed.argtypes = [sz, U8P, U32P, U32P, U32P]
        L_.dev_ed448g_sum.argtypes = [sz, sz, U32P, U32P]
        L_.dev_ed448g_norm.argtypes = [ctypes.c_int, sz, sz, U32P, ctypes.c_void_p]
        L_.dev_ed448g_error_string.restype = ctypes.c_char_p
        assert L_.dev_ed448g_is_device() == (1 if kind == "device" else 0)
        g = (ctypes.c_int * 6)()
        L_.dev_ed448g_geometry(g)
        self.block, self.minblk, self.fb_minblk, self.fbw, self.fbnd, self.fb_words = list(g)

    def ok(self, rc):
        assert rc == 0, f"rc {rc}: {self.lib.dev_ed448g_error_string(rc).decode()}"

    def scalar_ok(self, recs):
        inp = _arr(recs)
        out = np.zeros(len(recs), np.uint8)
        self.ok(self.lib.dev_ed448g_scalar_ok(len(recs), _p(inp, U8P), _p(out, U8P)))
        return [int(v) for v in out]

    def decompress(self, recs):
        inp = _arr(recs)
        xy, fl = np.zeros(28 * len(recs), np.uint32), np.zeros(len(recs), np.uint8)
        self.ok(self.lib.dev_ed448g_decompress(len(recs), _p(inp, U8P), _p(xy, U32P), _p(fl, U8P)))
        return [int(f) for f in fl], xy

    def mul(self, ks57, ps57, ct=False):
        """-> (extended points as SoA words, status words)"""
        n = len(ks57)
        k = _arr(ks57)
        p = _arr(ps57) if ps57 is not None else None
        ext, st = np.zeros(56 * n, np.uint32), np.zeros(2, np.uint32)
        self.ok(self.lib.dev_ed448g_mul(n, _p(k, U8P), _p(p, U8P) if p is not None else None, int(ct), _p(ext, U32P), _p(st, U32P)))
        return ext, [int(st[0]), int(st[1])]

    def fixed(self, ks57, table):
        n = len(ks57)
        k = _arr(ks57)
        ext, st = np.zeros(56 * n, np.uint32), np.zeros(2, np.uint32)
        self.ok(self.lib.dev_ed448g_fixed(n, _p(k, U8P), _p(table, U32P), _p(ext, U32P), _p(st, U32P)))
        return ext, [int(st[0]), int(st[1])]

    def sum(self, ext, n_in, n_out):
        out = np.zeros(56 * n_out, np.uint32)
        self.ok(self.lib.dev_ed448g_sum(n_in, n_out, _p(ext, U32P), _p(out, U32P)))
        return out

    def norm(self, ext, n, threads, table=False):
        out = np.zeros(n * (168 if table else 57), np.uint8)
        self.ok(self.lib.dev_ed448g_norm(1 if table else 0, n, threads, _p(ext, U32P), out.ctypes.data))
        return out


def _p(a, t):
    return a.ctypes.data_as(t)


def _arr(recs):
    return np.frombuffer(b"".join(recs), np.uint8).copy()


def ext_points(ext, n):
    """SoA words -> [(X, Y, Z, T)] integers"""
    w = np.asarray(ext, np.uint32).reshape(56, n)
    out = []
    for i in range(n):
        col = w[:, i]
        vals = [int.from_bytes(col[14 * c:14 * c + 14].tobytes(), "little") for c in range(4)]
        out.append(vals)
    return out


def to_soa(pts):
    """[(X, Y, Z, T)] integers -> SoA words"""
    n = len(pts)
    w = np.zeros((56, n), np.uint32)
    for i, p in enumerate(pts):
        for c in range(4):
            w[14 * c:14 * c + 14, i] = np.frombuffer(p[c].to_bytes(56, "little"), np.uint32)
    return w.reshape(-1).copy()


def affine(e):
    X, Y, Z, T = e
    assert T * Z % P == X * Y % P  # T = XY/Z
    zi = M.inv(Z)
    return X * zi % P, Y * zi % P


_BACKENDS = {}


def backend(kind):
    if kind not in _BACKENDS:
        _BACKENDS[kind] = GroupDev(kind)
    return _BACKENDS[kind]


@pytest.fixture(scope="module", params=[pytest.param("host", id="host"), pytest.param("device", id="device", marks=pytest.mark.gpu)])
def be(request):
    return backend(request.param)


def test_dev_scalar_check(be):
    recs = [G.enc_scalar(v, b) for v in (0, 1, 2, L - 1, L, L + 1, 2**446 - 1, 2**446, 2**448 - 1) for b in (0, 1, 0x80, 0xFF)]
    recs += [random.Random(i).getrandbits(446 + (i % 3)).to_bytes(56, "little") + bytes([i & 0xFF]) for i in range(200)]
    assert be.scalar_ok(recs) == [int(G.scalar_ok(r)) for r in recs]


def group_decompress_cases():
    rng = random.Random(487)
    recs = []
    for y in (0, 1, 2, P - 1, P, P + 1, 2**448 - 1):
        for sign in (0, 1):
            for low in (0, 0x2A, 0x7F):
                recs.append(enc_y(y, sign, low))
    for i in range(24):
        pt = rand_point(rng)
        for T in (M.IDENTITY,) + M.TORSION:
            e = bytearray(M.encode(M.add(pt, T)))
            e[56] |= i & 0x7F
            recs.append(bytes(e))
    recs += [enc_y(rng.getrandbits(448), rng.getrandbits(1)) for _ in range(60)]
    recs += [bytes.fromhex(v["public"]) for v in GOLDEN["vectors"]] + [bytes(57), ID]
    return recs


def test_dev_group_decompress(be):
    """flag bit 1 is the group decoder (the identity accepted under both sign bits, (0, -1) and the all-zero record
    refused); bit 0 and (x, y) are ed448_decode's"""
    recs = group_decompress_cases()
    flags, raw = be.decompress(recs)
    for r, f in zip(recs, flags):
        pt = M.decompress_unchecked(r)
        assert (f & 1) == (pt is not None), r.hex()
        assert (f >> 1) == (G.decompress(r) is not None), r.hex()
    ids = [i for i, r in enumerate(recs) if G.decompress(r) == M.IDENTITY]
    assert len(ids) >= 8 and all(flags[i] == 3 for i in ids)  # the verification predicate would refuse these
    assert flags[recs.index(bytes(57))] == 1  # decodes (order 4), refused
    if be.kind == "device":
        assert np.array_equal(raw, backend("host").decompress(recs)[1])


def test_dev_mul_var_edge_scalars(be):
    """the variable-base kernel over edge scalars on random subgroup points, the identity and B (P57 = NULL), default
    and constant-time paths bit-identical"""
    rng = random.Random(5)
    ks = edge_scalars()
    pts = [rand_point(rng) for _ in range(5)] + [M.IDENTITY]
    pairs = [(k, pts[i % len(pts)]) for i, k in enumerate(ks)]
    k57 = [G.enc_scalar(k, 0xFF if i % 7 == 0 else 0) for i, (k, _) in enumerate(pairs)]
    p57 = [M.encode(p) for _, p in pairs]
    ext, st = be.mul(k57, p57)
    assert st == [0, 0xFFFFFFFF]
    got = [affine(e) for e in ext_points(ext, len(pairs))]
    assert got == [M.mul(k, p) for k, p in pairs]
    ext_ct, _ = be.mul(k57, p57, ct=True)
    assert np.array_equal(ext, ext_ct)
    extb, _ = be.mul(k57[:40], None)
    assert [affine(e) for e in ext_points(extb, 40)] == [M.mul(k, M.B) for k, _ in pairs[:40]]
    if be.kind == "device":
        assert np.array_equal(ext, backend("host").mul(k57, p57)[0])


def test_dev_mul_reports_refusals(be):
    k57 = [G.enc_scalar(3)] * 8
    p57 = [M.encode(M.B)] * 8
    k57[5] = G.enc_scalar(L)
    p57[6] = enc_y(P - 1)
    _, st = be.mul(k57, p57)
    assert st == [3, 5]
    k57[5] = G.enc_scalar(1)
    _, st = be.mul(k57, p57)
    assert st == [2, 6]
    p57[6] = bytes(57)
    p57[2] = M.encode(M.add(M.B, M.TORSION[0]))
    _, st = be.mul(k57, p57)
    assert st == [2, 2]


@pytest.fixture(scope="module")
def model_table():
    g = backend("host")
    return np.frombuffer(G.fixed_base_table(g.fbw, g.fbnd), np.uint32).copy()


def test_dev_fixed_base(be, model_table):
    """the fixed-base accumulation over a table built by the model"""
    assert model_table.size == be.fb_words
    ks = edge_scalars()
    k57 = [G.enc_scalar(k) for k in ks]
    ext, st = be.fixed(k57, model_table)
    assert st == [0, 0xFFFFFFFF]
    assert [affine(e) for e in ext_points(ext, len(ks))] == [M.mul(k, M.B) for k in ks]
    _, st = be.fixed([G.enc_scalar(1), G.enc_scalar(L + 5), G.enc_scalar(2**447)], model_table)
    assert st == [1, 1]
    if be.kind == "device":
        assert np.array_equal(ext, backend("host").fixed(k57, model_table)[0])


def test_dev_normalise_and_compress(be):
    """Montgomery's trick along strided slices (1, several and one element per thread), a slice with the identity, and
    the table-entry form"""
    rng = random.Random(9)
    pts = [rand_point(rng)]
    for _ in range(600):
        pts.append(M.add(pts[-1], M.B))
    pts += [M.IDENTITY, M.B, M.neg(M.B)]
    pts[7] = pts[300] = M.IDENTITY
    exts = []
    for pt in pts:
        z = rng.randrange(1, P)
        exts.append([pt[0] * z % P, pt[1] * z % P, z, pt[0] * pt[1] * z % P])
    soa = to_soa(exts)
    n = len(pts)
    want = b"".join(M.encode(p) for p in pts)
    for threads in (1, 129, n):  # whole blocks of 128 threads: slices of 5, 3 and 1 elements
        assert be.norm(soa, n, threads).tobytes() == want, threads
    tab = be.norm(soa, n, 1, table=True).tobytes()
    assert tab == b"".join(x.to_bytes(56, "little") + y.to_bytes(56, "little") + (M.D * x * y % P).to_bytes(56, "little") for x, y in pts)
    assert M.encode(M.IDENTITY) == ID


def test_dev_sum(be):
    rng = random.Random(31)
    pts = [rand_point(rng) for _ in range(70)] + [M.IDENTITY]
    exts = []
    for pt in pts:
        z = rng.randrange(1, P)
        exts.append([pt[0] * z % P, pt[1] * z % P, z, pt[0] * pt[1] * z % P])
    soa = to_soa(exts)
    n = len(pts)
    for n_out in (1, 3, 32):
        parts = [affine(e) for e in ext_points(be.sum(soa, n, n_out), n_out)]
        for t in range(n_out):
            acc = M.IDENTITY
            for i in range(t, n, n_out):
                acc = M.add(acc, pts[i])
            assert parts[t] == acc


# ---- the C ABI, the Python and C++ mirrors ----------------------------------------------------------------------------------
def test_abi_null_ctx():
    import ecgpu

    lib = ecgpu.load_library()
    z = np.zeros(128, np.uint8)
    assert lib.ecg_ed448_mul_batch(None, 1, z.ctypes.data, z.ctypes.data, z.ctypes.data) == ecgpu.ECG_EINVAL
    assert lib.ecg_ed448_mul_gen_batch(None, 1, z.ctypes.data, z.ctypes.data) == ecgpu.ECG_EINVAL
    assert lib.ecg_ed448_lincomb(None, 1, z.ctypes.data, z.ctypes.data, z.ctypes.data) == ecgpu.ECG_EINVAL
    assert lib.ecg_ed448_lincomb(None, 0, None, None, None) == ecgpu.ECG_EINVAL


CPP = r"""
#include "ecgpu.hpp"
#include <cstdio>
int main() {
  try {
    ecgpu::Engine eng(ECG_SECP256K1);
    std::vector<ecgpu::Engine::Ed448Scalar> k(3);
    k[0][0] = 1;
    k[1][0] = 2;
    auto b = eng.ed448_mul_gen(k);
    std::vector<ecgpu::Engine::Ed448Point> P = {b[0], b[0], b[1]};
    auto m = eng.ed448_mul(k, P);
    auto s = eng.ed448_lincomb(k, P);
    auto e = eng.ed448_lincomb({}, {});
    std::printf("gen=%%d mul=%%d lin=%%d id=%%d\n", (int)(b[0][0] == 0x14 && b[2][0] == 1), (int)(m[1] == b[1] && m[2][0] == 1),
                (int)(s == eng.ed448_mul_gen({ecgpu::Engine::Ed448Scalar{3}})[0]), (int)(e[0] == 1 && e[56] == 0));
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


def test_cpp_mirror_ed448_group_compiles_and_links():
    import torch

    rc, out = _cpp_run()
    if torch.cuda.is_available():
        assert rc == 0, out
    else:
        assert rc == 42, out  # ECG_ECUDA without a GPU


@pytest.mark.gpu
def test_cpp_mirror_ed448_group_for_real():
    rc, out = _cpp_run()
    assert rc == 0, out
    assert "gen=1 mul=1 lin=1 id=1" in out


@pytest.fixture(scope="module")
def eng():
    import ecgpu

    e = ecgpu.Engine([0])
    yield e
    e.close()


def seeds(n, seed):
    rng = random.Random(seed)
    return [rng.getrandbits(456).to_bytes(57, "little") for _ in range(n)]


def recs(ks, byte56=0):
    return _arr([G.enc_scalar(k, byte56) for k in ks])


def rows(a):
    return [bytes(r) for r in np.asarray(a).reshape(-1, 57)]


@pytest.fixture(scope="module")
def keyset():
    """2^16 seeds with their clamped secret scalars (mod ell) and OpenSSL's public keys"""
    ss = seeds(1 << 16, 65536)
    return ss, [G.secret_scalar(s) for s in ss], [openssl_public(s) for s in ss]


@pytest.mark.gpu
def test_abi_mul_gen_openssl(eng, keyset):
    ss, a, pubs = keyset
    got = rows(eng.ed448_mul_gen(recs(a)))
    assert got == pubs
    for v in GOLDEN["vectors"]:
        assert bytes(eng.ed448_mul_gen(recs([G.secret_scalar(bytes.fromhex(v["seed"]))]))[0]).hex() == v["public"]


@pytest.mark.gpu
def test_abi_mul_cross_check(eng, keyset):
    """mul(k, pub(s)) == mul_gen(k a(s) mod ell) over 2^16 pairs; a 512-element sample against the model; [ell - k]P is
    -[k]P (byte 56 differs in bit 7 alone, unless x = 0)"""
    ss, a, pubs = keyset
    rng = random.Random(7)
    ks = [rng.randrange(L) for _ in ss]
    ks[:6] = [0, 1, 2, L - 1, L - 2, 4]
    got = eng.ed448_mul(recs(ks), _arr(pubs))
    want = eng.ed448_mul_gen(recs([k * ai % L for k, ai in zip(ks, a)]))
    assert np.array_equal(got, want)
    for i in range(512):
        assert bytes(got[i]) == G.mul(G.enc_scalar(ks[i]), pubs[i]), i
    neg = eng.ed448_mul(recs([(L - k) % L for k in ks[:4096]]), _arr(pubs[:4096]))
    for i in range(4096):
        g, n = bytes(got[i]), bytes(neg[i])
        assert g[:56] == n[:56]
        x_zero = g == ID
        assert n[56] == (g[56] if x_zero else g[56] ^ 0x80)


@pytest.mark.gpu
def test_abi_rejected_inputs(eng):
    import ecgpu

    n = 300
    k = recs([5] * n)
    P_ = _arr([M.encode(M.B)] * n)
    assert rows(eng.ed448_mul(k, P_))[0] == M.encode(M.mul(5, M.B))
    cases = [(10, "k", G.enc_scalar(L)), (11, "k", G.enc_scalar(2**446, 0xFF)), (12, "P", enc_y(P - 1)), (13, "P", bytes(57)),
             (14, "P", M.encode(M.add(M.B, M.TORSION[1]))), (15, "P", enc_y(non_decodable_y()))]
    for idx, what, rec in cases:
        for first in (idx, 250):
            kk, pp = k.copy(), P_.copy()
            for j in (first, 299):
                (kk if what == "k" else pp)[57 * j:57 * j + 57] = np.frombuffer(rec, np.uint8)
            err = ecgpu.ScalarRangeError if what == "k" else ecgpu.NotOnCurveError
            with pytest.raises(err) as ei:
                eng.ed448_mul(kk, pp)
            assert ei.value.index == first
            if what == "k":
                with pytest.raises(err) as ei:
                    eng.ed448_mul_gen(kk)
                assert ei.value.index == first
            with pytest.raises(err) as ei:
                eng.ed448_lincomb(kk, pp)
            assert ei.value.index == first
    # byte 56 = 0xFF with a small scalar is accepted and gives the same output as byte 56 = 0
    assert np.array_equal(eng.ed448_mul(recs([5] * 4, 0xFF), P_[:228]), eng.ed448_mul(recs([5] * 4), P_[:228]))
    assert np.array_equal(eng.ed448_mul_gen(recs([5, 7], 0xFF)), eng.ed448_mul_gen(recs([5, 7])))


@pytest.mark.gpu
def test_abi_identity_in_and_out(eng):
    idents = [ID, enc_y(1, 1), enc_y(1, 1, 0x7F), enc_y(P + 1)]
    out = rows(eng.ed448_mul(recs([0, 1, 2, L - 1]), _arr(idents)))
    assert out == [ID] * 4
    out = rows(eng.ed448_mul(recs([0, L - 1, 1]), _arr([M.encode(M.B)] * 3)))
    assert out == [ID, M.encode(M.neg(M.B)), M.encode(M.B)]
    assert rows(eng.ed448_mul_gen(recs([0, 1, L - 1]))) == [ID, M.encode(M.B), M.encode(M.neg(M.B))]


@pytest.mark.gpu
def test_abi_lincomb_small(eng):
    """n = 0, 1, 2, 57 (the shape of the reference's test_pow_add_mul) and 1,000 terms against the model"""
    assert bytes(eng.ed448_lincomb(np.zeros(0, np.uint8), np.zeros(0, np.uint8))) == ID
    rng = random.Random(57)
    for n in (1, 2, 57, 1000):
        pts = [M.encode(rand_point(rng)) if i % 9 else ID for i in range(n)]
        ks = [rng.randrange(L) if i % 5 else [0, 1, L - 1, 2, 3][i // 5 % 5] for i in range(n)]
        got = bytes(eng.ed448_lincomb(recs(ks), _arr(pts)))
        assert got == G.lincomb([G.enc_scalar(k) for k in ks], pts), n
    # P + (-P) = O
    b, nb = M.encode(M.B), M.encode(M.neg(M.B))
    assert bytes(eng.ed448_lincomb(recs([3, 3]), _arr([b, nb]))) == ID


@pytest.mark.gpu
def test_abi_lincomb_algebraic(eng, keyset):
    """sum k_i [s_i]B == [sum k_i s_i mod ell]B over 2^16 terms"""
    ss, a, pubs = keyset
    rng = random.Random(16)
    ks = [rng.randrange(L) for _ in ss]
    got = bytes(eng.ed448_lincomb(recs(ks), _arr(pubs)))
    want = bytes(eng.ed448_mul_gen(recs([sum(k * ai for k, ai in zip(ks, a)) % L]))[0])
    assert got == want == G.mul_gen(G.enc_scalar(sum(k * ai for k, ai in zip(ks, a)) % L))


def _wave(minblk):
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count * minblk * 128


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["mul", "mul_gen"])
def test_abi_ragged_sizes(eng, which):
    """sizes across the host chunks (a wave is sm_count * 2 * 128 elements), n = 0"""
    n0 = _wave(2)
    rng = random.Random(n0)
    base = [M.encode(rand_point(rng)) for _ in range(8)]
    for n in (0, 1, 129, 2 * n0 + 5, 4 * n0 + 3):
        ks = [rng.randrange(L) for _ in range(n)]
        if which == "mul":
            pts = [base[i % 8] for i in range(n)]
            out = eng.ed448_mul(recs(ks) if n else np.zeros(0, np.uint8), _arr(pts) if n else np.zeros(0, np.uint8))
            idx = range(0, n, max(1, n // 40))
            for i in idx:
                assert bytes(out[i]) == G.mul(G.enc_scalar(ks[i]), pts[i]), (n, i)
            if n:
                assert bytes(out[-1]) == G.mul(G.enc_scalar(ks[-1]), pts[-1])
        else:
            out = eng.ed448_mul_gen(recs(ks) if n else np.zeros(0, np.uint8))
            ct = __import__("ecgpu").Engine([0], consttime=True)
            assert np.array_equal(out, ct.ed448_mul_gen(recs(ks) if n else np.zeros(0, np.uint8)))
            ct.close()
            for i in list(range(0, n, max(1, n // 40))) + ([n - 1] if n else []):
                assert bytes(out[i]) == G.mul_gen(G.enc_scalar(ks[i])), (n, i)


@pytest.mark.gpu
def test_abi_device_pointers():
    import torch

    import ecgpu

    rng = random.Random(99)
    n = 4099
    ks = [rng.randrange(L) for _ in range(n)]
    pts = [M.encode(rand_point(rng)) for _ in range(16)]
    pts = [pts[i % 16] for i in range(n)]
    h = ecgpu.Engine([0])
    want_mul, want_gen = h.ed448_mul(recs(ks), _arr(pts)), h.ed448_mul_gen(recs(ks))
    want_lin = h.ed448_lincomb(recs(ks), _arr(pts))
    h.close()
    e = ecgpu.Engine([0], device_ptrs=True)
    # records at odd addresses: they are read and written bytewise
    kd = torch.zeros(57 * n + 1, dtype=torch.uint8, device="cuda")
    kd[1:] = torch.from_numpy(recs(ks)).cuda()
    pd = torch.zeros(57 * n + 3, dtype=torch.uint8, device="cuda")
    pd[3:] = torch.from_numpy(_arr(pts)).cuda()
    od = torch.zeros(57 * n + 1, dtype=torch.uint8, device="cuda")
    launches = e.kernel_launches
    e.ed448_mul_ptr(n, kd.data_ptr() + 1, pd.data_ptr() + 3, od.data_ptr() + 1)
    torch.cuda.synchronize()
    assert e.kernel_launches == launches + 2  # the scalar multiplication and the normalisation
    assert np.array_equal(od[1:].cpu().numpy(), want_mul.reshape(-1))
    e.ed448_mul_gen_ptr(n, kd.data_ptr() + 1, od.data_ptr() + 1)
    torch.cuda.synchronize()
    assert np.array_equal(od[1:].cpu().numpy(), want_gen.reshape(-1))
    o1 = torch.zeros(58, dtype=torch.uint8, device="cuda")
    e.ed448_lincomb_ptr(n, kd.data_ptr() + 1, pd.data_ptr() + 3, o1.data_ptr() + 1)
    torch.cuda.synchronize()
    assert np.array_equal(o1[1:].cpu().numpy(), want_lin)
    e.ed448_lincomb_ptr(0, 0, 0, o1.data_ptr() + 1)
    torch.cuda.synchronize()
    assert bytes(o1[1:].cpu().numpy()) == ID
    bad = kd.clone()
    bad[1 + 57 * 7:1 + 57 * 7 + 56] = 0xFF
    with pytest.raises(ecgpu.ScalarRangeError) as ei:
        e.ed448_mul_ptr(n, bad.data_ptr() + 1, pd.data_ptr() + 3, od.data_ptr() + 1)
    assert ei.value.index == 7
    e.close()


@pytest.mark.gpu
def test_abi_consttime_and_zeroize_identical(eng):
    import ecgpu

    rng = random.Random(2051)
    n = 2051
    ks = [rng.randrange(L) for _ in range(n)]
    ks[:4] = [0, 1, 2, L - 1]
    pts = [M.encode(rand_point(rng)) for _ in range(8)] + [ID]
    pts = [pts[i % 9] for i in range(n)]
    base = (eng.ed448_mul(recs(ks), _arr(pts)), eng.ed448_mul_gen(recs(ks)), eng.ed448_lincomb(recs(ks), _arr(pts)))
    for kw in ({"zeroize": True}, {"consttime": True}, {"zeroize": True, "consttime": True}):
        e = ecgpu.Engine([0], **kw)
        got = (e.ed448_mul(recs(ks), _arr(pts)), e.ed448_mul_gen(recs(ks)), e.ed448_lincomb(recs(ks), _arr(pts)))
        for g, b in zip(got, base):
            assert np.array_equal(g, b), kw
        e.close()


@pytest.mark.gpu
def test_abi_timing_brackets_the_kernel(eng):
    rng = random.Random(4)
    ks = recs([rng.randrange(L) for _ in range(4096)])
    P_ = _arr([M.encode(M.B)] * 4096)
    for call in (lambda: eng.ed448_mul(ks, P_), lambda: eng.ed448_mul_gen(ks), lambda: eng.ed448_lincomb(ks, P_)):
        eng.timing_enable(True)
        call()
        ms, calls = eng.timing_read()
        eng.timing_enable(False)
        assert calls == 1 and ms > 0


@pytest.mark.gpu
def test_abi_einval(eng):
    import ecgpu

    lib, c = eng.lib, eng._ctx
    z, ids = np.zeros(57 * 2, np.uint8), _arr([ID, ID])
    d = z.ctypes.data
    assert lib.ecg_ed448_mul_batch(c, 2, d, ids.ctypes.data, d) == ecgpu.ECG_OK
    for args in ((None, d, d), (d, None, d), (d, d, None)):
        assert lib.ecg_ed448_mul_batch(c, 2, *args) == ecgpu.ECG_EINVAL
        assert lib.ecg_ed448_lincomb(c, 2, *args) == ecgpu.ECG_EINVAL
    assert lib.ecg_ed448_mul_gen_batch(c, 2, None, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_ed448_mul_gen_batch(c, 2, d, None) == ecgpu.ECG_EINVAL
    assert lib.ecg_ed448_mul_batch(c, 0, None, None, None) == ecgpu.ECG_OK
    assert lib.ecg_ed448_mul_gen_batch(c, 0, None, None) == ecgpu.ECG_OK
    assert lib.ecg_ed448_lincomb(c, 0, None, None, d) == ecgpu.ECG_OK
    assert lib.ecg_ed448_lincomb(c, 0, None, None, None) == ecgpu.ECG_EINVAL
    assert bytes(z[:57]) == ID


@pytest.mark.gpu
def test_abi_multi_device():
    import torch

    import ecgpu

    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    rng = random.Random(2)
    n = 5003
    ks = [rng.randrange(L) for _ in range(n)]
    pts = [M.encode(rand_point(rng)) for _ in range(8)]
    pts = [pts[i % 8] for i in range(n)]
    one, two = ecgpu.Engine([0]), ecgpu.Engine([0, 1])
    assert np.array_equal(one.ed448_mul(recs(ks), _arr(pts)), two.ed448_mul(recs(ks), _arr(pts)))
    assert np.array_equal(one.ed448_mul_gen(recs(ks)), two.ed448_mul_gen(recs(ks)))
    assert np.array_equal(one.ed448_lincomb(recs(ks), _arr(pts)), two.ed448_lincomb(recs(ks), _arr(pts)))
    one.close()
    two.close()
