"""Ed448 verification (RFC 8032): the Python model, the device pieces (SHAKE256, scalars mod ell, decompression, the
subgroup test, the group, the per-signature routine) as the kernel compiles them, and ecg_ed448_verify_batch through the
C ABI, the Python mirror and the C++ mirror.

Oracles: the reference's own vectors (tests/golden/ed448.json: RFC 8032 sections 7.4-7.5, the negative cases of its
test, the compressed generator and ell), OpenSSL's Ed448 through `cryptography`, hashlib's SHAKE256 and the model in
ed448_model.py (Python integers).  The device library (tests/dev/ed448_dev.cu, under the kernel's launch bound) runs
under the `gpu` marker; its host twin runs everywhere, and the device must give its bits.

Where the reference and OpenSSL disagree the reference wins (test_documented_disagreements): a y >= p in A or R is
reduced, bits 0-6 of byte 56 of A or R are ignored by decompression but hashed as given, and S = 0 is refused."""
import ctypes
import json
import multiprocessing as mp
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

import ed448_model as M

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = os.path.join(HERE, "dev")
LIB = os.path.join(ROOT, "elliptic-curves_b200", "libecgpu.so")
GOLDEN = json.load(open(os.path.join(HERE, "golden", "ed448.json")))
U8P = ctypes.POINTER(ctypes.c_uint8)
U32P = ctypes.POINTER(ctypes.c_uint32)
U64P = ctypes.POINTER(ctypes.c_uint64)
P, L = M.P, M.L


def _b(h):
    return bytes.fromhex(h)


def openssl_verify(pk: bytes, sig: bytes, msg: bytes) -> bool:
    from cryptography.exceptions import InvalidSignature
    from cryptography.hazmat.primitives.asymmetric.ed448 import Ed448PublicKey

    try:
        Ed448PublicKey.from_public_bytes(pk).verify(sig, msg)
        return True
    except (InvalidSignature, ValueError):
        return False


def openssl_keypair(seed: bytes):
    from cryptography.hazmat.primitives.asymmetric.ed448 import Ed448PrivateKey

    sk = Ed448PrivateKey.from_private_bytes(seed)
    return sk, sk.public_key().public_bytes_raw()


def vector_cases():
    """(pk, sig, msg, ctx, prehashed, expected) for the six RFC vectors and the reference's negative cases"""
    out = []
    for v in GOLDEN["vectors"]:
        pk, sig, ctx, ph = _b(v["public"]), _b(v["sig"]), _b(v["ctx"]), v["prehashed"]
        msg = M.prehash(_b(v["msg"])) if ph else _b(v["msg"])
        out.append((pk, sig, msg, ctx, ph, True))
        out.append((pk, sig, msg, _b(GOLDEN["negatives"]["wrong_context"]), ph, False))
        if ph:
            f = GOLDEN["negatives"]["prehash_flip"]
            bad = bytearray(msg)
            bad[f["byte"]] ^= f["xor"]
            out.append((pk, sig, bytes(bad), ctx, ph, False))
        else:
            out.append((pk, sig, _b(GOLDEN["negatives"]["wrong_message"]), ctx, ph, False))
    return out


def enc_y(y: int, sign: int = 0, low: int = 0) -> bytes:
    """57-byte encoding of y (any integer below 2^448) with the sign bit and bits 0-6 of byte 56"""
    return y.to_bytes(56, "little") + bytes([(sign << 7) | low])


def small_subgroup_y():
    """the smallest y whose point lies in the prime-order subgroup (y + p < 2^448: a non-canonical encoding exists)"""
    y = 2
    while True:
        pt = M.decompress(enc_y(y))
        if pt is not None:
            return y
        y += 1


def non_residue_y(n):
    """y values whose (1 - y^2) / (1 - d y^2) has no square root"""
    out, y = [], 2
    while len(out) < n:
        if M.decompress_unchecked(enc_y(y)) is None:
            out.append(y)
        y += 1
    return out


def torsioned(pk: bytes):
    """the encodings of A + T for the three torsion points T other than the identity"""
    A = M.decompress(pk)
    return [M.encode(M.add(A, T)) for T in M.TORSION]


def corrupt_cases(n, seed):
    """model- and OpenSSL-made cases: n keys with messages of 0 .. 300 bytes, each signature valid or corrupted (a
    flipped bit in R, S, A or M; S + ell; S with byte 56 set; A the identity; A or R plus a torsion point; a y with no
    square root; S = 0).  -> (pk, sig, msg)"""
    rng = random.Random(seed)
    cases = []
    nr = non_residue_y(8)
    for i in range(n):
        sk, pk = openssl_keypair(rng.getrandbits(456).to_bytes(57, "little"))
        msg = bytes(rng.getrandbits(8) for _ in range(rng.randrange(301)))
        sig = sk.sign(msg)
        kind = i % 13
        s = bytearray(sig)
        if kind == 1:
            s[rng.randrange(56)] ^= 1 << rng.randrange(8)  # R, not byte 56
        elif kind == 2:
            s[57 + rng.randrange(56)] ^= 1 << rng.randrange(8)
        elif kind == 3:
            p2 = bytearray(pk)
            p2[rng.randrange(56)] ^= 1 << rng.randrange(8)
            pk = bytes(p2)
        elif kind == 4 and msg:
            m2 = bytearray(msg)
            m2[rng.randrange(len(msg))] ^= 1 << rng.randrange(8)
            msg = bytes(m2)
        elif kind == 5:
            sv = int.from_bytes(sig[57:113], "little") + L
            s[57:113] = sv.to_bytes(56, "little")
        elif kind == 6:
            s[113] = 1
        elif kind == 7:
            pk = M.encode(M.IDENTITY)
        elif kind == 8:
            pk = torsioned(pk)[i % 3]
        elif kind == 9:
            s[:57] = torsioned(sig[:57])[i % 3]
        elif kind == 10:
            pk = enc_y(nr[i % 8], i & 1)
        elif kind == 11:
            s[57:] = bytes(57)  # S = 0
        cases.append((pk, bytes(s), msg))
    return cases


def _model_verdicts(cases):
    return [M.verify(pk, sig, msg) for pk, sig, msg in cases]


def model_many(cases, ctx=b"", prehashed=False):
    """the model's verdicts, over the host cores"""
    if ctx or prehashed:
        return [M.verify(pk, sig, msg, ctx, prehashed) for pk, sig, msg in cases]
    procs = min(os.cpu_count() or 1, 32)
    step = max(1, (len(cases) + procs * 4 - 1) // (procs * 4))
    with mp.Pool(procs) as pool:
        parts = pool.map(_model_verdicts, [cases[i:i + step] for i in range(0, len(cases), step)])
    return [v for p in parts for v in p]


# ---- the model ----------------------------------------------------------------------------------------------------------
def test_golden_constants():
    assert int(GOLDEN["order"], 16) == L
    assert M.encode(M.B) == _b(GOLDEN["generator"]) == M.B_BYTES
    assert M.mul(L, M.B) == M.IDENTITY


def test_generated_header():
    """ecg_ed448_consts.cuh is exactly what tools/gen_ed448_consts.py derives from the public parameters, and its base
    table holds the odd multiples of the model's B"""
    import importlib.util

    spec = importlib.util.spec_from_file_location("gen_ed448_consts", os.path.join(ROOT, "tools", "gen_ed448_consts.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    with open(os.path.join(ROOT, "elliptic-curves_b200", "csrc", "ecg_ed448_consts.cuh")) as f:
        assert f.read() == gen.render()
    assert (gen.BX, gen.BY) == M.B and gen.L == L and gen.D == M.D


def test_model_reproduces_rfc_vectors():
    for v in GOLDEN["vectors"]:
        seed, ctx, ph = _b(v["seed"]), _b(v["ctx"]), v["prehashed"]
        msg = M.prehash(_b(v["msg"])) if ph else _b(v["msg"])
        assert M.public_key(seed).hex() == v["public"]
        assert M.sign(seed, msg, ctx, ph).hex() == v["sig"]
    for pk, sig, msg, ctx, ph, want in vector_cases():
        assert M.verify(pk, sig, msg, ctx, ph) == want


def test_fast_subgroup_predicate():
    """the device's predicate on y equals [ell]P == O on subgroup points, their torsion translates, and random points"""
    rng = random.Random(1164)
    for _ in range(40):
        pt = M.mul(rng.randrange(1, L), M.B)
        for T in (M.IDENTITY,) + M.TORSION:
            q = M.add(pt, T)
            assert M.torsion_free_fast(q[1]) == M.torsion_free(q)
    for _ in range(200):
        pt = M.decompress_unchecked(enc_y(rng.getrandbits(448) % P))
        if pt is not None:
            assert M.torsion_free_fast(pt[1]) == M.torsion_free(pt)
    for T in (M.IDENTITY,) + M.TORSION:
        assert M.torsion_free_fast(T[1]) == (T == M.IDENTITY)


def test_model_against_openssl():
    cases = corrupt_cases(1024, seed=8032)
    got = model_many(cases)
    for (pk, sig, msg), g in zip(cases, got):
        assert g == openssl_verify(pk, sig, msg), (pk.hex(), sig.hex(), msg.hex())
    assert 0 < sum(got) < len(got)


def test_documented_disagreements():
    """the reference accepts what OpenSSL refuses (non-canonical A / R bytes that the signer hashed as given) and refuses
    S = 0; y >= p decodes to the point of y - p"""
    seed = bytes(range(57))
    _, pk = openssl_keypair(seed)
    msg = b"non-canonical"
    for low in (1, 0x40, 0x7F):
        pk_nc = pk[:56] + bytes([pk[56] | low])
        sig = M.sign(seed, msg, pk=pk_nc)
        assert M.verify(pk_nc, sig, msg) and not openssl_verify(pk_nc, sig, msg)
        sig_r = M.sign(seed, msg, r_bytes_of=lambda rb: rb[:56] + bytes([rb[56] | low]))
        assert M.verify(pk, sig_r, msg) and not openssl_verify(pk, sig_r, msg)
    sig = M.sign(seed, msg)
    assert M.verify(pk, sig, msg)
    assert not M.verify(pk, sig[:57] + bytes(57), msg)  # S = 0
    y = small_subgroup_y()
    assert M.decompress(enc_y(y + P)) == M.decompress(enc_y(y)) is not None


# ---- device library and its host twin -----------------------------------------------------------------------------------
class Ed448Dev:
    def __init__(self, kind):
        import __graft_entry__ as ge

        ge.build()
        self.kind = kind
        L_ = self.lib = ctypes.CDLL(os.path.join(DEV, "libecged448dev.so" if kind == "device" else "libecged448devsim.so"))
        L_.dev_ed448_shake.argtypes = [ctypes.c_size_t, U8P, ctypes.c_size_t, U64P, U8P]
        L_.dev_ed448_mod_l.argtypes = [ctypes.c_size_t, U8P, U32P]
        L_.dev_ed448_s_ok.argtypes = [ctypes.c_size_t, U8P, U8P]
        L_.dev_ed448_decompress.argtypes = [ctypes.c_size_t, U8P, U32P, U8P]
        L_.dev_ed448_point.argtypes = [ctypes.c_int, ctypes.c_size_t, U32P, U32P]
        L_.dev_ed448_verify.argtypes = [ctypes.c_size_t, U8P, U8P, U8P, ctypes.c_size_t, U64P, U8P, ctypes.c_uint32, U8P]
        L_.dev_ed448_error_string.restype = ctypes.c_char_p
        assert L_.dev_ed448_is_device() == (1 if kind == "device" else 0)

    def ok(self, rc):
        assert rc == 0, f"rc {rc}: {self.lib.dev_ed448_error_string(rc).decode()}"

    @staticmethod
    def packed(msgs):
        offs = np.zeros(len(msgs) + 1, np.uint64)
        offs[1:] = np.cumsum([len(m) for m in msgs])
        data = np.frombuffer(b"".join(msgs) + b"\0", np.uint8).copy()
        return data, offs

    def shake(self, msgs):
        data, offs = self.packed(msgs)
        out = np.zeros(114 * len(msgs), np.uint8)
        self.ok(self.lib.dev_ed448_shake(len(msgs), _p(data, U8P), data.size - 1, _p(offs, U64P), _p(out, U8P)))
        return [out[114 * i:114 * i + 114].tobytes() for i in range(len(msgs))]

    def mod_l(self, vals):
        inp = np.frombuffer(b"".join(v.to_bytes(114, "little") for v in vals), np.uint8).copy()
        out = np.zeros(14 * len(vals), np.uint32)
        self.ok(self.lib.dev_ed448_mod_l(len(vals), _p(inp, U8P), _p(out, U32P)))
        return [int.from_bytes(out[14 * i:14 * i + 14].tobytes(), "little") for i in range(len(vals))]

    def s_ok(self, recs):
        inp = np.frombuffer(b"".join(recs), np.uint8).copy()
        out = np.zeros(len(recs), np.uint8)
        self.ok(self.lib.dev_ed448_s_ok(len(recs), _p(inp, U8P), _p(out, U8P)))
        return list(out)

    def decompress(self, recs):
        inp = np.frombuffer(b"".join(recs), np.uint8).copy()
        xy, fl = np.zeros(28 * len(recs), np.uint32), np.zeros(len(recs), np.uint8)
        self.ok(self.lib.dev_ed448_decompress(len(recs), _p(inp, U8P), _p(xy, U32P), _p(fl, U8P)))
        v = [int.from_bytes(xy[14 * j:14 * j + 14].tobytes(), "little") for j in range(2 * len(recs))]
        return [(int(fl[i]), v[2 * i], v[2 * i + 1]) for i in range(len(recs))], xy

    def point(self, op, rows):
        inp = np.frombuffer(b"".join(x.to_bytes(56, "little") for r in rows for x in r), np.uint32).copy()
        out = np.zeros(56 * len(rows), np.uint32)
        self.ok(self.lib.dev_ed448_point(op, len(rows), _p(inp, U32P), _p(out, U32P)))
        v = [int.from_bytes(out[14 * j:14 * j + 14].tobytes(), "little") for j in range(4 * len(rows))]
        return [v[4 * i:4 * i + 4] for i in range(len(rows))], out

    def verify(self, cases, ctx=b"", prehashed=False):
        n = len(cases)
        pk = np.frombuffer(b"".join(c[0] for c in cases), np.uint8).copy()
        sig = np.frombuffer(b"".join(c[1] for c in cases), np.uint8).copy()
        data, offs = self.packed([c[2] for c in cases])
        dom = np.frombuffer(M.dom4(1 if prehashed else 0, ctx), np.uint8).copy()
        valid = np.zeros(n, np.uint8)
        self.ok(self.lib.dev_ed448_verify(n, _p(pk, U8P), _p(sig, U8P), _p(data, U8P), data.size - 1, _p(offs, U64P), _p(dom, U8P),
                                          dom.size, _p(valid, U8P)))
        return list(valid)


def _p(a, t):
    return a.ctypes.data_as(t)


_BACKENDS = {}


def backend(kind):
    if kind not in _BACKENDS:
        _BACKENDS[kind] = Ed448Dev(kind)
    return _BACKENDS[kind]


@pytest.fixture(scope="module", params=[pytest.param("host", id="host"), pytest.param("device", id="device", marks=pytest.mark.gpu)])
def be(request):
    return backend(request.param)


def test_shake256(be):
    rng = random.Random(256)
    msgs = [bytes(rng.getrandbits(8) for _ in range(n)) for n in (0, 1, 135, 136, 137, 271, 272, 273, 1000)]
    assert be.shake(msgs) == [M.shake256(m) for m in msgs]


def test_mod_l(be):
    rng = random.Random(446)
    vals = [0, L - 1, L, L + 1, 2 * L, 2 * L - 1, 2**446 - 1, 2**446, 2**448 - 1, 2**896 - 1, 2**912 - 1]
    vals += [rng.getrandbits(912) for _ in range(500)] + [rng.getrandbits(rng.randrange(1, 913)) for _ in range(500)]
    assert be.mod_l(vals) == [v % L for v in vals]


def test_s_check(be):
    recs = [v.to_bytes(56, "little") + b"\0" for v in (0, 1, 2, L - 1, L, L + 1, 2**446 - 1, 2**448 - 1)]
    recs += [(1).to_bytes(56, "little") + bytes([b]) for b in (1, 0x80, 0xFF)]
    recs += [random.Random(i).getrandbits(446).to_bytes(56, "little") + b"\0" for i in range(100)]
    assert be.s_ok(recs) == [int(M.s_ok(r)) for r in recs]


def decompress_cases():
    y0 = small_subgroup_y()
    recs = []
    for y in (0, 1, 2, P - 1, P, P + 1, 2**448 - 1, y0, y0 + P) + tuple(non_residue_y(6)):
        for sign in (0, 1):
            for low in (0, 1, 0x55, 0x7F):
                recs.append(enc_y(y, sign, low))
    rng = random.Random(57)
    for i in range(40):
        pt = M.mul(rng.randrange(1, L), M.B)
        for T in (M.IDENTITY,) + M.TORSION:
            e = bytearray(M.encode(M.add(pt, T)))
            e[56] |= i & 0x7F
            recs.append(bytes(e))
    recs += [enc_y(rng.getrandbits(448), rng.getrandbits(1)) for _ in range(100)]
    recs += [_b(GOLDEN["generator"])] + [_b(v["public"]) for v in GOLDEN["vectors"]]
    return recs


def test_decompress(be):
    recs = decompress_cases()
    got, raw = be.decompress(recs)
    accepted = 0
    for r, (fl, x, y) in zip(recs, got):
        pt = M.decompress_unchecked(r)
        assert (fl & 1) == (pt is not None), r.hex()
        if pt is None:
            assert fl == 0
            continue
        assert (x, y) == pt, r.hex()
        want = M.decompress(r) is not None and pt != M.IDENTITY
        assert (fl >> 1) == want, r.hex()
        accepted += want
    assert accepted > 40
    if be.kind == "device":
        assert np.array_equal(raw, backend("host").decompress(recs)[1])


def ext(pt, z):
    """affine -> extended coordinates scaled by z"""
    x, y = pt
    return [x * z % P, y * z % P, z % P, x * y * z % P]


def test_point_ops(be):
    """dbl and add on extended inputs (Z != 1, torsion points, the identity, P + (-P), P + P) against the model; a
    chain of 64 steps through the device's own outputs"""
    rng = random.Random(448)
    pts = [M.mul(rng.randrange(1, L), M.B) for _ in range(24)] + list(M.TORSION) + [M.IDENTITY, M.B]
    dbl_rows = [ext(p, rng.randrange(1, P)) for p in pts]
    add_pairs = [(p, q) for p in pts[:10] for q in pts[20:]] + [(p, M.neg(p)) for p in pts[:5]] + [(p, p) for p in pts[:5]]
    add_rows = [ext(p, rng.randrange(1, P)) + ext(q, rng.randrange(1, P)) for p, q in add_pairs]

    def aff(r):
        zi = M.inv(r[2])
        assert r[3] * r[2] % P == r[0] * r[1] % P  # T Z == X Y
        return r[0] * zi % P, r[1] * zi % P

    got, raw_d = be.point(0, dbl_rows)
    assert [aff(r) for r in got] == [M.add(p, p) for p in pts]
    got, raw_a = be.point(1, add_rows)
    assert [aff(r) for r in got] == [M.add(p, q) for p, q in add_pairs]
    # chain: Q <- 2 Q + B, 64 times, through the device's raw outputs
    q, want = ext(pts[0], 7), pts[0]
    for _ in range(64):
        (d,), _ = be.point(0, [q])
        (q,), _ = be.point(1, [d + ext(M.B, 1)])
        want = M.add(M.add(want, want), M.B)
    assert aff(q) == want
    if be.kind == "device":
        assert np.array_equal(raw_d, backend("host").point(0, dbl_rows)[1])
        assert np.array_equal(raw_a, backend("host").point(1, add_rows)[1])


def test_verify_one(be):
    """the whole per-signature routine through the kernel: the RFC vectors and their negatives, OpenSSL-signed
    corrupted cases, model-made contexts, Ed448ph and the non-canonical encodings the reference accepts"""
    for pk, sig, msg, ctx, ph, want in vector_cases():
        assert be.verify([(pk, sig, msg)], ctx, ph) == [int(want)]
    cases = corrupt_cases(260, seed=57)
    want = model_many(cases)
    got = be.verify(cases)
    assert got == [int(w) for w in want]
    assert 0 < sum(got) < len(got)
    seed = bytes(57)
    _, pk = openssl_keypair(seed)
    ctx = b"context" * 36  # 252 bytes
    mctx = [(pk, M.sign(seed, m, ctx), m) for m in (b"", b"a" * 200)]
    assert be.verify(mctx, ctx) == [1, 1] and be.verify(mctx, ctx[:-1]) == [0, 0]
    mph = [(pk, M.sign(seed, M.prehash(m), b"", True), M.prehash(m)) for m in (b"", b"abc")]
    assert be.verify(mph, b"", True) == [1, 1] and be.verify(mph) == [0, 0]
    nc = [(pk[:56] + bytes([pk[56] | 0x7F]), M.sign(seed, b"x", pk=pk[:56] + bytes([pk[56] | 0x7F])), b"x"),
          (pk, M.sign(seed, b"y", r_bytes_of=lambda rb: rb[:56] + bytes([rb[56] | 3])), b"y")]
    assert be.verify(nc) == [1, 1]
    if be.kind == "device":
        assert got == backend("host").verify(cases)


# ---- the C ABI, the Python and C++ mirrors ------------------------------------------------------------------------------
def test_abi_null_ctx():
    import ecgpu

    lib = ecgpu.load_library()
    z = np.zeros(128, np.uint8)
    o = np.zeros(2, np.uint64)
    assert lib.ecg_ed448_verify_batch(None, 1, z.ctypes.data, z.ctypes.data, z.ctypes.data, o.ctypes.data, None, 0, 0,
                                      z.ctypes.data) == ecgpu.ECG_EINVAL
    assert lib.ecg_ed448_verify_batch(None, 0, None, None, None, None, None, 0, 0, None) == ecgpu.ECG_EINVAL


CPP = r"""
#include "ecgpu.hpp"
#include <cstdio>
static void unhex(const char* h, uint8_t* out, size_t n) {
  for (size_t i = 0; i < n; i++) {
    unsigned b;
    std::sscanf(h + 2 * i, "%%2x", &b);
    out[i] = (uint8_t)b;
  }
}
int main() {
  try {
    ecgpu::Engine eng(ECG_SECP256K1);
    std::vector<ecgpu::Engine::Ed448Key> pk(2);
    std::vector<ecgpu::Engine::Ed448Sig> sig(2);
    unhex("%(pk)s", pk[0].data(), 57);
    unhex("%(sig)s", sig[0].data(), 114);
    pk[1] = pk[0];
    sig[1] = sig[0];
    std::vector<std::vector<uint8_t>> msgs = {{0x03}, {0x04}};
    auto v = eng.ed448_verify(pk, sig, msgs);
    auto w = eng.ed448_verify(pk, sig, msgs, {0x66, 0x6f, 0x6f});
    std::printf("valid=%%d%%d ctx=%%d%%d\n", (int)v[0], (int)v[1], (int)w[0], (int)w[1]);
    return 0;
  } catch (const ecgpu::Error& e) {
    std::printf("error %%d\n", (int)e.code);
    return e.code == ECG_ECUDA ? 42 : 3;  // 42: no GPU -> a loud failure, no CPU fallback
  }
}
"""


def _cpp_run():
    v = GOLDEN["vectors"][1]  # 1-byte message 03, empty context
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "e.cpp"), os.path.join(d, "e")
        open(src, "w").write(CPP % {"pk": v["public"], "sig": v["sig"]})
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "elliptic-curves_b200", "host"), src, LIB,
                               "-Wl,-rpath," + os.path.dirname(LIB), "-o", exe])
        p = subprocess.run([exe], capture_output=True, text=True, timeout=300)
        return p.returncode, p.stdout + p.stderr


def test_cpp_mirror_ed448_compiles_and_links():
    import torch

    rc, out = _cpp_run()
    if torch.cuda.is_available():
        assert rc == 0, out
    else:
        assert rc == 42, out  # ECG_ECUDA without a GPU


@pytest.mark.gpu
def test_cpp_mirror_ed448_for_real():
    rc, out = _cpp_run()
    assert rc == 0, out
    assert "valid=10 ctx=00" in out


@pytest.fixture(scope="module")
def eng():
    import ecgpu

    e = ecgpu.Engine([0])
    yield e
    e.close()


def _arr(recs):
    return np.frombuffer(b"".join(recs), np.uint8).copy()


def _run(e, cases, ctx=b"", ph=False):
    return list(e.ed448_verify(_arr([c[0] for c in cases]), _arr([c[1] for c in cases]), [c[2] for c in cases], ctx, ph))


@pytest.mark.gpu
def test_abi_rfc_vectors_all_modes(eng):
    """Ed448 (empty context), Ed448 with a context, Ed448ph, with the reference's negative cases"""
    for pk, sig, msg, ctx, ph, want in vector_cases():
        assert _run(eng, [(pk, sig, msg)], ctx, ph) == [int(want)], (pk.hex(), ctx, ph)


def openssl_batch(n, seed, msg_len=64):
    """n OpenSSL signatures over msg_len-byte messages from 64 keys, a quarter of them corrupted by one flipped bit in R,
    S, A or M (bytes 0..55 of R and A, so that the encodings stay canonical) -> (cases, OpenSSL's verdicts)"""
    rng = random.Random(seed)
    keys = [openssl_keypair(rng.getrandbits(456).to_bytes(57, "little")) for _ in range(64)]
    cases, want = [], []
    for i in range(n):
        sk, pk = keys[i % 64]
        msg = rng.getrandbits(8 * msg_len).to_bytes(msg_len, "little")
        sig = bytearray(sk.sign(msg))
        if i % 4 == 3:
            where = (i // 4) % 4
            if where == 0:
                sig[rng.randrange(56)] ^= 1 << rng.randrange(8)
            elif where == 1:
                sig[57 + rng.randrange(56)] ^= 1 << rng.randrange(8)
            elif where == 2:
                p2 = bytearray(pk)
                p2[rng.randrange(56)] ^= 1 << rng.randrange(8)
                pk = bytes(p2)
            else:
                m2 = bytearray(msg)
                m2[rng.randrange(msg_len)] ^= 1 << rng.randrange(8)
                msg = bytes(m2)
        cases.append((pk, bytes(sig), msg))
        want.append(int(openssl_verify(pk, bytes(sig), msg)))
    return cases, want


@pytest.mark.gpu
def test_abi_openssl_batch(eng):
    n = 1 << 16
    cases, want = openssl_batch(n, seed=65536)
    got = _run(eng, cases)
    assert got == want
    assert sum(want) == n - n // 4  # every corruption is refused
    sample = cases[:512]
    assert got[:512] == [int(v) for v in model_many(sample)]


@pytest.mark.gpu
def test_abi_model_made(eng):
    """contexts, Ed448ph, the non-canonical encodings the reference accepts, S = 0 and y >= p"""
    seed = bytes(range(57))
    _, pk = openssl_keypair(seed)
    ctx = bytes(range(255))
    msgs = [b"", b"m" * 137, bytes(range(256))]
    assert _run(eng, [(pk, M.sign(seed, m, ctx), m) for m in msgs], ctx) == [1, 1, 1]
    ph = [M.prehash(m) for m in msgs]
    assert _run(eng, [(pk, M.sign(seed, h, b"foo", True), h) for h in ph], b"foo", True) == [1, 1, 1]
    assert _run(eng, [(pk, M.sign(seed, h, b"foo", True), h) for h in ph], b"foo", False) == [0, 0, 0]
    nc = []
    for low in (1, 0x2A, 0x7F):
        pk_nc = pk[:56] + bytes([pk[56] | low])
        nc.append((pk_nc, M.sign(seed, b"nc", pk=pk_nc), b"nc"))
        nc.append((pk, M.sign(seed, b"nc", r_bytes_of=lambda rb, low=low: rb[:56] + bytes([rb[56] | low])), b"nc"))
    assert _run(eng, nc) == [1] * 6
    good = M.sign(seed, b"s0")
    y = small_subgroup_y()
    odd = [(pk, good[:57] + bytes(57), b"s0"), (enc_y(y + P), good, b"s0"), (pk, enc_y(y + P) + good[57:], b"s0")]
    assert _run(eng, odd) == [int(M.verify(*c)) for c in odd] == [0, 0, 0]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 257, 2 * 132 * 2 * 128 + 5])
def test_abi_ragged_sizes(eng, n):
    """sizes across the host chunks (a wave is sm_count * 2 * 128 signatures), n = 0 and empty messages"""
    rng = random.Random(n)
    keys = [openssl_keypair(rng.getrandbits(456).to_bytes(57, "little")) for _ in range(16)]
    cases = []
    for i in range(n):
        sk, pk = keys[i % 16]
        msg = b"" if i % 3 == 0 else rng.getrandbits(8 * (i % 50)).to_bytes(i % 50, "little")
        sig = sk.sign(msg)
        cases.append((pk, sig if i % 5 else sig[:-2] + b"\1\0", msg))
    if n == 0:
        v = eng.ed448_verify(np.zeros(0, np.uint8), np.zeros(0, np.uint8), [])
        assert v.shape == (0,)
        return
    got = _run(eng, cases)
    assert got == [int(openssl_verify(*c)) for c in cases]


@pytest.mark.gpu
def test_abi_device_pointers():
    import torch

    import ecgpu

    cases, want = openssl_batch(4099, seed=99)
    data, offs = ecgpu.Engine._pack_messages([c[2] for c in cases])
    e = ecgpu.Engine([0], device_ptrs=True)
    pkd = torch.from_numpy(_arr([c[0] for c in cases])).cuda()
    sgd = torch.from_numpy(_arr([c[1] for c in cases])).cuda()
    md = torch.from_numpy(data).cuda()
    od = torch.from_numpy(offs.view(np.int64)).cuda()
    vd = torch.zeros(len(cases), dtype=torch.uint8, device="cuda")
    launches = e.kernel_launches
    e.ed448_verify_ptr(len(cases), pkd.data_ptr(), sgd.data_ptr(), md.data_ptr(), od.data_ptr(), vd.data_ptr())
    torch.cuda.synchronize()
    assert e.kernel_launches == launches + 1
    assert list(vd.cpu().numpy()) == want
    # records at odd addresses: they are read bytewise
    pk1 = torch.zeros(57 * len(cases) + 1, dtype=torch.uint8, device="cuda")
    pk1[1:] = pkd
    vd.zero_()
    e.ed448_verify_ptr(len(cases), pk1.data_ptr() + 1, sgd.data_ptr(), md.data_ptr(), od.data_ptr(), vd.data_ptr())
    torch.cuda.synchronize()
    assert list(vd.cpu().numpy()) == want
    # offsets not 8-byte aligned, decreasing offsets
    o2 = torch.zeros(len(cases) + 2, dtype=torch.int64, device="cuda")
    o2[1:] = od
    with pytest.raises(ecgpu.EcgError):
        e.ed448_verify_ptr(len(cases), pkd.data_ptr(), sgd.data_ptr(), md.data_ptr(), o2.data_ptr() + 4, vd.data_ptr())
    bad = od.clone()
    bad[5] = bad[6] + 1
    with pytest.raises(ecgpu.EcgError):
        e.ed448_verify_ptr(len(cases), pkd.data_ptr(), sgd.data_ptr(), md.data_ptr(), bad.data_ptr(), vd.data_ptr())
    e.close()


@pytest.mark.gpu
def test_abi_zeroize_and_consttime_flags(eng):
    import ecgpu

    cases, want = openssl_batch(2051, seed=2051)
    for kw in ({"zeroize": True}, {"consttime": True}, {"zeroize": True, "consttime": True}):
        e = ecgpu.Engine([0], **kw)
        assert _run(e, cases) == want, kw
        e.close()


@pytest.mark.gpu
def test_abi_timing_brackets_the_kernel(eng):
    cases, _ = openssl_batch(4096, seed=4)
    eng.timing_enable(True)
    _run(eng, cases)
    ms, calls = eng.timing_read()
    eng.timing_enable(False)
    assert calls == 1 and ms > 0


@pytest.mark.gpu
def test_abi_einval(eng):
    import ecgpu

    lib, c = eng.lib, eng._ctx
    pk, sig = np.zeros(57 * 2, np.uint8), np.zeros(114 * 2, np.uint8)
    msgs, offs, valid = np.zeros(8, np.uint8), np.array([0, 4, 8], np.uint64), np.zeros(2, np.uint8)
    ctx = np.zeros(256, np.uint8)
    d = lambda a: a.ctypes.data  # noqa: E731

    def call(n=2, pk_=d(pk), sig_=d(sig), m=d(msgs), o=d(offs), cx=None, cl=0, v=d(valid)):
        return lib.ecg_ed448_verify_batch(c, n, pk_, sig_, m, o, cx, cl, 0, v)

    assert call() == ecgpu.ECG_OK
    for kw in ({"pk_": None}, {"sig_": None}, {"o": None}, {"v": None}, {"m": None}, {"cl": 256, "cx": d(ctx)}, {"cl": 3}):
        assert call(**kw) == ecgpu.ECG_EINVAL, kw
    assert call(o=d(np.array([0, 5, 4], np.uint64))) == ecgpu.ECG_EINVAL
    assert call(cl=255, cx=d(ctx)) == ecgpu.ECG_OK
    assert call(n=0, pk_=None, sig_=None, m=None, o=None, v=None) == ecgpu.ECG_OK
    assert call(m=None, o=d(np.zeros(3, np.uint64))) == ecgpu.ECG_OK  # every message empty
    with pytest.raises(ecgpu.EcgError):
        eng.ed448_verify(pk, sig, [b"", b""], context=bytes(256))


@pytest.mark.gpu
def test_abi_multi_device():
    import torch

    import ecgpu

    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    cases, want = openssl_batch(5003, seed=2)
    e = ecgpu.Engine([0, 1])
    assert _run(e, cases) == want
    e.close()
