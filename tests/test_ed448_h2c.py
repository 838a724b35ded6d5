"""Ed448 hash to curve (RFC 9380 edwards448_XOF:SHAKE256_ELL2_RO_ / _NU_) and hash to scalar: the model
(ed448_h2c_model.py) against the reference's vectors, and its reference-literal formulas against the device's
straight-line ones; the device routines (tests/dev/ed448_h2c_dev.cu: the 84-byte reductions, the map with the isogeny,
uniform bytes to compressed points through the normalisation kernel, the hash kernels, under the production launch
bounds) against their host twin and the model; the ecg_ed448_hash_* entries through the C ABI, the Python and C++
mirrors.

Oracles: the reference's RO and NU vectors, its hash_to_field (from_okm) vectors under the curve448 and edwards448 DSTs
and its scalar_hash vector (tests/golden/ed448_h2c.json, extracted by tools/extract_ed448_h2c_golden.py), and the
reference's formulas restated in Python."""
import ctypes
import json
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

import ed448_group_model as G
import ed448_h2c_model as H
import ed448_model as M

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = os.path.join(HERE, "dev")
LIB = os.path.join(ROOT, "elliptic-curves_b200", "libecgpu.so")
GOLDEN = json.load(open(os.path.join(HERE, "golden", "ed448_h2c.json")))
U8P = ctypes.POINTER(ctypes.c_uint8)
U32P = ctypes.POINTER(ctypes.c_uint32)
U64P = ctypes.POINTER(ctypes.c_uint64)
P, L = M.P, M.L
RO, NU = H.HASH_TO_CURVE_ID, H.ENCODE_TO_CURVE_ID
ZERO = H.ZERO_RECORD
EXCEPTIONAL = (0, 1, P - 1)


def be84(v: int) -> bytes:
    return v.to_bytes(84, "big")


def golden_points(key):
    """the DST and (message, first, second) of a fixture table: affine x, y, or hash_to_field's u0, u1"""
    g = GOLDEN[key]
    a, b = ("u0", "u1") if key.startswith("from_okm") else ("x", "y")
    return bytes.fromhex(g["dst"]), [(bytes.fromhex(v["msg"]), int(v[a], 16), int(v[b], 16)) for v in g["vectors"]]


def branch_us():
    """u forcing each (e2, sgn0 of the root found) combination, found by search in the model"""
    rng = random.Random(44)
    want, found = {(a, b) for a in (True, False) for b in (0, 1)}, {}
    while set(found) != want:
        u = rng.randrange(2, P - 1)
        _, _, _, e2, s = H.dev_map_parts(u)
        found.setdefault((e2, s), u)
    return [found[k] for k in sorted(found)]


# ---- the model ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key,nu", [("hash_to_curve", False), ("encode_to_curve", True)])
def test_model_vectors(key, nu):
    """the reference's RO / NU vectors: affine (x, y), through the reference-literal and the device formulas"""
    dst, vecs = golden_points(key)
    for msg, x, y in vecs:
        want = M.encode((x, y))
        assert M.on_curve((x, y)) and M.torsion_free((x, y))
        assert H.hash_to_curve(msg, dst, nu) == want
        assert H.hash_to_curve(msg, dst, nu, device_form=True) == want


@pytest.mark.parametrize("key", ["from_okm_curve448", "from_okm_edwards448"])
def test_model_hash_to_field(key):
    """expand_message_xof to 168 bytes, each 84-byte block big-endian mod p (little-endian reading fails)"""
    dst, vecs = golden_points(key)
    for msg, u0, u1 in vecs:
        assert H.hash_to_field(msg, dst) == (u0, u1)
        u = H.expand_message_xof(msg, dst, 168)
        assert int.from_bytes(u[:84], "little") % P != u0


def test_model_scalar_hash():
    sh = GOLDEN["scalar_hash"]
    assert H.hash_to_scalar(bytes.fromhex(sh["msg"]), bytes.fromhex(sh["dst"])).hex() == sh["scalar"]


def test_model_forms_agree():
    """reference-literal and straight-line map agree on random u, on every (e2, sgn0) branch and on the exceptional u;
    the isogeny's images are curve points except at (0, 0)"""
    rng = random.Random(9380)
    us = [rng.randrange(P) for _ in range(300)] + branch_us() + [2, P - 2, P - 3]
    for u in us:
        e = H.dev_map(u)
        x, y = H.ref_isogeny(H.ref_map(u))
        assert e[2] != 0 and (e[0] * M.inv(e[2]) % P, e[1] * M.inv(e[2]) % P) == (x, y), u
        assert M.on_curve((x, y))
        assert e[3] * e[2] % P == e[0] * e[1] % P
    for u0, u1 in zip(us[:100], us[100:200]):
        assert H.compress_ext(H.ref_point(u0, u1)) == H.compress_ext(H.dev_point(u0, u1))
        assert H.compress_ext(H.ref_point(u0)) == H.compress_ext(H.dev_point(u0))


def test_model_exceptional_u():
    """u in {0, 1, p - 1}: the reference maps to (0, 0) and outputs 57 zero bytes in NU and in RO with either half
    exceptional; the device form gives (0 : 0 : 0 : 0) and the same bytes; 1 - A and -A are not squares"""
    assert not M.is_square(1 - H.A) and not M.is_square(-H.A)
    for u in EXCEPTIONAL:
        assert H.ref_map(u) == (0, 0) and H.ref_isogeny((0, 0)) == (0, 0)
        assert H.dev_map(u) == (0, 0, 0, 0)
        assert H.compress_ext(H.ref_point(u)) == ZERO == H.compress_ext(H.dev_point(u))
        for v in (5, 1, u):
            assert H.compress_ext(H.ref_point(u, v)) == ZERO == H.compress_ext(H.dev_point(u, v))
            assert H.compress_ext(H.ref_point(v, u)) == ZERO == H.compress_ext(H.dev_point(v, u))
    assert H.compress_ext(H.ref_point(5)) != ZERO


def test_model_empty_dst():
    with pytest.raises(ValueError):
        H.hash_to_curve(b"x", b"")


# ---- device library and its host twin ------------------------------------------------------------------------------------
class H2cDev:
    def __init__(self, kind):
        import __graft_entry__ as ge

        ge.build()
        self.kind = kind
        L_ = self.lib = ctypes.CDLL(os.path.join(DEV, "libecged448h2cdev.so" if kind == "device" else "libecged448h2cdevsim.so"))
        sz = ctypes.c_size_t
        L_.dev_edh_load84.argtypes = [sz, U8P, U32P]
        L_.dev_edh_mod_l_84.argtypes = [sz, U8P, U8P]
        L_.dev_edh_map.argtypes = [sz, U32P, U32P]
        L_.dev_edh_from_uniform.argtypes = [sz, U8P, ctypes.c_int, U32P, U8P]
        L_.dev_edh_hash.argtypes = [sz, U8P, U64P, U8P, ctypes.c_uint32, ctypes.c_int, U8P]
        L_.dev_edh_error_string.restype = ctypes.c_char_p
        assert L_.dev_edh_is_device() == (1 if kind == "device" else 0)

    def ok(self, rc):
        assert rc == 0, f"rc {rc}: {self.lib.dev_edh_error_string(rc).decode()}"

    def load84(self, bs):
        out = np.zeros(14 * len(bs), np.uint32)
        self.ok(self.lib.dev_edh_load84(len(bs), _p(_arr(bs), U8P), _p(out, U32P)))
        return [int.from_bytes(out[14 * i:14 * i + 14].tobytes(), "little") for i in range(len(bs))]

    def mod_l_84(self, bs):
        out = np.zeros(57 * len(bs), np.uint8)
        self.ok(self.lib.dev_edh_mod_l_84(len(bs), _p(_arr(bs), U8P), _p(out, U8P)))
        return _rows(out)

    def map(self, us):
        n = len(us)
        u14 = np.frombuffer(b"".join(u.to_bytes(56, "little") for u in us), np.uint32).copy()
        ext = np.zeros(56 * n, np.uint32)
        self.ok(self.lib.dev_edh_map(n, _p(u14, U32P), _p(ext, U32P)))
        return ext_points(ext, n)

    def from_uniform(self, us):
        n, ln = len(us), len(us[0])
        ext, out = np.zeros(56 * n, np.uint32), np.zeros(57 * n, np.uint8)
        self.ok(self.lib.dev_edh_from_uniform(n, _p(_arr(us), U8P), ln, _p(ext, U32P), _p(out, U8P)))
        return ext_points(ext, n), _rows(out)

    def hash(self, msgs, suffix, mode):
        offs = np.zeros(len(msgs) + 1, np.uint64)
        offs[1:] = np.cumsum([len(m) for m in msgs])
        data = np.frombuffer(b"".join(msgs) + b"\0", np.uint8).copy()
        sfx = np.frombuffer(suffix, np.uint8).copy()
        out = np.zeros(57 * len(msgs), np.uint8)
        self.ok(self.lib.dev_edh_hash(len(msgs), _p(data, U8P), _p(offs, U64P), _p(sfx, U8P), len(suffix), mode, _p(out, U8P)))
        return _rows(out)


def _p(a, t):
    return a.ctypes.data_as(t)


def _arr(recs):
    return np.frombuffer(b"".join(recs), np.uint8).copy()


def _rows(a):
    return [bytes(r) for r in np.asarray(a, np.uint8).reshape(-1, 57)]


def ext_points(ext, n):
    w = np.asarray(ext, np.uint32).reshape(56, n)
    return [[int.from_bytes(w[14 * c:14 * c + 14, i].tobytes(), "little") for c in range(4)] for i in range(n)]


_BACKENDS = {}


def backend(kind):
    if kind not in _BACKENDS:
        _BACKENDS[kind] = H2cDev(kind)
    return _BACKENDS[kind]


@pytest.fixture(scope="module", params=[pytest.param("host", id="host"), pytest.param("device", id="device", marks=pytest.mark.gpu)])
def be(request):
    return backend(request.param)


def reduction_edges():
    """0, p - 1, p, 2p, 2^448 - 1, 2^672 - 1, values whose high 224 bits fold across 2^224 with carries, random"""
    vals = [0, 1, P - 1, P, P + 1, 2 * P, 2 * P - 1, 2**448 - 1, 2**448, 2**672 - 1, 2**672 - 2**448, (2**224 - 1) << 448,
            ((2**224 - 1) << 448) | (2**448 - 1), ((2**224 - 1) << 448) | (2**224 - 1) << 224, (1 << 448) | (2**224 - 1) << 224,
            (P << 224) % 2**672, 2**671]
    rng = random.Random(84)
    vals += [rng.getrandbits(672) for _ in range(200)]
    return [be84(v) for v in vals]


def test_dev_load84(be):
    bs = reduction_edges()
    got = be.load84(bs)
    assert all(g < 2**448 for g in got)
    assert [g % P for g in got] == [H.reduce84(b) for b in bs]


def test_dev_mod_l_84(be):
    vals = [0, 1, L - 1, L, L + 1, 2 * L, 2**672 - 1, 2**446, 2**448 - 1, 2**671]
    rng = random.Random(57)
    vals += [rng.getrandbits(672) for _ in range(200)]
    bs = [be84(v) for v in vals]
    assert be.mod_l_84(bs) == [H.reduce84_scalar(b) for b in bs]
    assert be.mod_l_84([be84(L - 1)])[0] == (L - 1).to_bytes(57, "little")


def test_dev_map(be):
    """the map with the homogenised isogeny on random u, every branch and the exceptional u (also as non-canonical
    limbs: p and p + 1), and 2^448 - 1"""
    rng = random.Random(441)
    us = EXCEPTIONAL + (P, P + 1, 2**448 - 1) + tuple(branch_us()) + tuple(rng.randrange(P) for _ in range(100))
    got = be.map(list(us))
    for u, e in zip(us, got):
        want = H.dev_map(u % P)
        if u % P in EXCEPTIONAL:
            assert [c % P for c in e] == [0, 0, 0, 0], u
            continue
        x, y = H.ref_isogeny(H.ref_map(u % P))
        zi = M.inv(e[2])
        assert (e[0] * zi % P, e[1] * zi % P) == (x, y), u
        assert e[3] * e[2] % P == e[0] * e[1] % P
        assert [c % P for c in e] == list(want)


@pytest.mark.parametrize("ln", [84, 168])
def test_dev_from_uniform(be, ln):
    """uniform bytes -> compressed through the hash kernel's body and the normalisation kernel; 300 elements, so that a
    normalisation slice holds several, with exceptional blocks at 5, 140 and 299: their 57 zero bytes and the slices
    around them (one Z = 0 without the Z mask would zero its whole slice)"""
    rng = random.Random(ln)
    us = [bytes(rng.getrandbits(8) for _ in range(ln)) for _ in range(300)]
    blocks = {5: be84(1), 140: be84(2 * P - 1), 299: be84(0)}  # u = 1, p - 1 (read from 2p - 1) and 0
    for i, blk in blocks.items():
        us[i] = blk if ln == 84 else (us[i][:84] + blk if i == 299 else blk + us[i][84:])
    us[7] = be84(2**672 - 1) * (ln // 84)
    ext, got = be.from_uniform(us)
    want = [H.ref_from_uniform(u) for u in us]
    assert got == want
    assert [i for i, r in enumerate(got) if r == ZERO] == [5, 140, 299]
    for i in (5, 140, 299):
        assert ext[i][2] % P == 1 and ext[i][0] % P == 0 and ext[i][1] % P == 0


def test_dev_hash_kernels(be):
    """the production hash kernels over message lengths around the 136-byte SHAKE256 rate and DSTs of 1, 255 and 256
    bytes (the last one oversize)"""
    rng = random.Random(12)
    msgs = [bytes(rng.getrandbits(8) for _ in range(n)) for n in (0, 1, 135, 136, 137, 271, 272, 273)]
    msgs += [b"abc", b"hello world"]
    for dst in (b"Q", bytes(range(255)), bytes(range(256))):
        assert be.hash(msgs, H.xof_suffix(dst, 168), 0) == [H.hash_to_curve(m, dst) for m in msgs]
        assert be.hash(msgs, H.xof_suffix(dst, 84), 1) == [H.hash_to_curve(m, dst, True) for m in msgs]
        assert be.hash(msgs, H.xof_suffix(dst, 84), 2) == [H.hash_to_scalar(m, dst) for m in msgs]
    for key, mode, ln in (("hash_to_curve", 0, 168), ("encode_to_curve", 1, 84)):
        dst, vecs = golden_points(key)
        assert be.hash([m for m, _, _ in vecs], H.xof_suffix(dst, ln), mode) == [M.encode((x, y)) for _, x, y in vecs]
    if be.kind == "device":
        h = backend("host")
        for mode, ln in ((0, 168), (1, 84), (2, 84)):
            assert be.hash(msgs, H.xof_suffix(RO, ln), mode) == h.hash(msgs, H.xof_suffix(RO, ln), mode)


# ---- the C ABI, the Python and C++ mirrors ----------------------------------------------------------------------------------
def test_abi_null_ctx():
    import ecgpu

    lib = ecgpu.load_library()
    z = np.zeros(128, np.uint8)
    o = np.zeros(2, np.uint64)
    d = z.ctypes.data
    assert lib.ecg_ed448_hash_to_curve_batch(None, 1, d, o.ctypes.data, d, 1, 0, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_ed448_hash_to_scalar_batch(None, 1, d, o.ctypes.data, d, 1, d) == ecgpu.ECG_EINVAL


CPP = r"""
#include "ecgpu.hpp"
#include <cstdio>
int main() {
  try {
    ecgpu::Engine eng(ECG_SECP256K1);
    std::vector<uint8_t> msg = {'h', 'e', 'l', 'l', 'o', ' ', 'w', 'o', 'r', 'l', 'd'};
    std::string d = "edwards448_XOF:SHAKE256_ELL2_RO_";
    std::vector<uint8_t> dst(d.begin(), d.end());
    auto hs = eng.ed448_hash_to_scalar({msg}, dst);
    auto hc = eng.ed448_hash_to_curve({msg, {}}, dst);
    auto hn = eng.ed448_hash_to_curve({msg}, dst, true);
    ecgpu::Engine::Ed448Scalar one{};
    one[0] = 1;
    auto m = eng.ed448_mul({one, hs[0]}, {hc[0], hc[1]});
    std::printf("h2s=%%02x%%02x%%02x top=%%d chain=%%d nu=%%d\n", hs[0][0], hs[0][1], hs[0][2], (int)hs[0][56], (int)(m[0] == hc[0]),
                (int)(hn[0] != hc[0]));
    return 0;
  } catch (const ecgpu::Error& e) {
    std::printf("error %%d\n", (int)e.code);
    return e.code == ECG_ECUDA ? 42 : 3;  // 42: no GPU -> a loud failure, no CPU fallback
  }
}
"""


def _cpp_run():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "h.cpp"), os.path.join(d, "h")
        open(src, "w").write(CPP % {})
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "elliptic-curves_b200", "host"), src, LIB,
                               "-Wl,-rpath," + os.path.dirname(LIB), "-o", exe])
        p = subprocess.run([exe], capture_output=True, text=True, timeout=300)
        return p.returncode, p.stdout + p.stderr


def test_cpp_mirror_ed448_h2c_compiles_and_links():
    import torch

    rc, out = _cpp_run()
    if torch.cuda.is_available():
        assert rc == 0, out
    else:
        assert rc == 42, out  # ECG_ECUDA without a GPU


@pytest.mark.gpu
def test_cpp_mirror_ed448_h2c_for_real():
    rc, out = _cpp_run()
    assert rc == 0, out
    assert "h2s=2d32a0 top=0 chain=1 nu=1" in out


@pytest.fixture(scope="module")
def eng():
    import ecgpu

    e = ecgpu.Engine([0])
    yield e
    e.close()


@pytest.mark.gpu
def test_abi_fixtures(eng):
    for key, nu in (("hash_to_curve", False), ("encode_to_curve", True)):
        dst, vecs = golden_points(key)
        assert _rows(eng.ed448_hash_to_curve([m for m, _, _ in vecs], dst, nonuniform=nu)) == [M.encode((x, y)) for _, x, y in vecs]
    sh = GOLDEN["scalar_hash"]
    assert bytes(eng.ed448_hash_to_scalar([bytes.fromhex(sh["msg"])], bytes.fromhex(sh["dst"]))[0]).hex() == sh["scalar"]


@pytest.mark.gpu
def test_abi_hash(eng):
    """RO, NU and hash to scalar on 4,096 messages of mixed lengths against the model under a short, a 255-byte and an
    oversize DST; the points are torsion free (ecg_ed448_mul_batch with k = 1 accepts them and returns the same bytes)
    and the scalars are accepted as scalars"""
    rng = random.Random(4096)
    lens = [0, 1, 135, 136, 137, 272, 1000] + [rng.randrange(0, 300) for _ in range(4089)]
    msgs = [bytes(rng.getrandbits(8) for _ in range(n)) for n in lens]
    one = _arr([G.enc_scalar(1)] * len(msgs))
    for dst in (RO, bytes(range(255)), bytes(range(256)) * 2):
        sample = range(0, 4096, 1 if dst == RO else 16)
        ro = _rows(eng.ed448_hash_to_curve(msgs, dst))
        nu = _rows(eng.ed448_hash_to_curve(msgs, dst, nonuniform=True))
        sc = _rows(eng.ed448_hash_to_scalar(msgs, dst))
        for i in sample:
            assert ro[i] == H.hash_to_curve(msgs[i], dst), i
            assert nu[i] == H.hash_to_curve(msgs[i], dst, True), i
            assert sc[i] == H.hash_to_scalar(msgs[i], dst), i
        for pts in (ro, nu):
            assert _rows(eng.ed448_mul(one, _arr(pts))) == pts
        gen = _rows(eng.ed448_mul_gen(_arr(sc)))
        for i in range(0, 4096, 512):
            assert gen[i] == G.mul_gen(sc[i]), i
        assert all(r[56] == 0 for r in sc)


@pytest.mark.gpu
def test_abi_einval(eng):
    import ecgpu

    lib, c = eng.lib, eng._ctx
    z = np.zeros(57 * 2, np.uint8)
    d = z.ctypes.data
    o = np.array([0, 1, 2], np.uint64)
    dst = np.frombuffer(RO, np.uint8).copy()
    for n in (0, 2):
        assert lib.ecg_ed448_hash_to_curve_batch(c, n, d, o.ctypes.data, dst.ctypes.data, 0, 0, d) == ecgpu.ECG_EINVAL  # EmptyDst
        assert lib.ecg_ed448_hash_to_curve_batch(c, n, d, o.ctypes.data, None, 5, 1, d) == ecgpu.ECG_EINVAL
        assert lib.ecg_ed448_hash_to_scalar_batch(c, n, d, o.ctypes.data, dst.ctypes.data, 0, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_ed448_hash_to_curve_batch(c, 2, d, None, dst.ctypes.data, dst.size, 0, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_ed448_hash_to_curve_batch(c, 2, d, o.ctypes.data, dst.ctypes.data, dst.size, 0, None) == ecgpu.ECG_EINVAL
    assert lib.ecg_ed448_hash_to_scalar_batch(c, 2, d, o.ctypes.data, dst.ctypes.data, dst.size, None) == ecgpu.ECG_EINVAL
    assert lib.ecg_ed448_hash_to_scalar_batch(c, 2, None, o.ctypes.data, dst.ctypes.data, dst.size, d) == ecgpu.ECG_EINVAL  # null msgs
    dec = np.array([0, 2, 1], np.uint64)
    assert lib.ecg_ed448_hash_to_curve_batch(c, 2, d, dec.ctypes.data, dst.ctypes.data, dst.size, 0, d) == ecgpu.ECG_EINVAL
    assert lib.ecg_ed448_hash_to_scalar_batch(c, 2, d, dec.ctypes.data, dst.ctypes.data, dst.size, d) == ecgpu.ECG_EINVAL
    empty = np.array([0, 0, 0], np.uint64)  # two empty messages need no message buffer
    assert lib.ecg_ed448_hash_to_curve_batch(c, 2, None, empty.ctypes.data, dst.ctypes.data, dst.size, 0, d) == ecgpu.ECG_OK
    assert _rows(z) == [H.hash_to_curve(b"", RO)] * 2
    big = np.zeros(300, np.uint8)  # n = 0: nothing launched, even for an oversize DST
    launches = eng.kernel_launches
    assert lib.ecg_ed448_hash_to_curve_batch(c, 0, None, None, big.ctypes.data, big.size, 0, None) == ecgpu.ECG_OK
    assert lib.ecg_ed448_hash_to_scalar_batch(c, 0, None, None, big.ctypes.data, big.size, None) == ecgpu.ECG_OK
    assert eng.kernel_launches == launches


def _wave(minblk):
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count * minblk * 128


@pytest.mark.gpu
def test_abi_ragged_sizes(eng):
    """sizes across the host chunks, n = 0"""
    n0 = _wave(2)
    for n in (0, 1, 129, 2 * n0 + 5, (1 << 18) + 3):
        msgs = [bytes([i & 0xFF]) * (i % 7) for i in range(n)]
        ro = _rows(eng.ed448_hash_to_curve(msgs, RO))
        sc = _rows(eng.ed448_hash_to_scalar(msgs, RO))
        assert len(ro) == len(sc) == n
        for i in list(range(0, n, max(1, n // 20))) + ([n - 1] if n else []):
            assert ro[i] == H.hash_to_curve(msgs[i], RO), (n, i)
            assert sc[i] == H.hash_to_scalar(msgs[i], RO), (n, i)


@pytest.mark.gpu
def test_abi_device_pointers():
    """device-resident messages, offsets and records at odd alignments; misaligned offsets are ECG_EINVAL"""
    import torch

    import ecgpu

    n = 4099
    msgs = [bytes([i & 0xFF]) * (i % 150) for i in range(n)]
    h = ecgpu.Engine([0])
    want = (h.ed448_hash_to_curve(msgs, RO), h.ed448_hash_to_curve(msgs, RO, True), h.ed448_hash_to_scalar(msgs, RO))
    h.close()
    e = ecgpu.Engine([0], device_ptrs=True)
    data, offs = ecgpu.Engine._pack_messages(msgs)
    dd = torch.zeros(data.size + 3, dtype=torch.uint8, device="cuda")
    dd[3:] = torch.from_numpy(data).cuda()
    do = torch.from_numpy(offs.view(np.int64)).cuda()
    od = torch.zeros(57 * n + 3, dtype=torch.uint8, device="cuda")
    for nu, w in ((False, want[0]), (True, want[1])):
        od.fill_(0xA5)
        e.ed448_hash_to_curve_ptr(n, dd.data_ptr() + 3, do.data_ptr(), od.data_ptr() + 3, RO, nu)
        torch.cuda.synchronize()
        assert np.array_equal(od[3:].cpu().numpy(), w.reshape(-1))
    e.ed448_hash_to_scalar_ptr(n, dd.data_ptr() + 3, do.data_ptr(), od.data_ptr() + 1, RO)
    torch.cuda.synchronize()
    assert np.array_equal(od[1:1 + 57 * n].cpu().numpy(), want[2].reshape(-1))
    # the records chain into the Ed448 group entry on the device: [1] P == P
    kd = torch.from_numpy(_arr([G.enc_scalar(1)] * n)).cuda()
    pd = torch.from_numpy(want[0].reshape(-1).copy()).cuda()
    o2 = torch.zeros(57 * n, dtype=torch.uint8, device="cuda")
    e.ed448_mul_ptr(n, kd.data_ptr(), pd.data_ptr(), o2.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(o2.cpu().numpy(), want[0].reshape(-1))
    od8 = torch.zeros(8 * (n + 2), dtype=torch.uint8, device="cuda")
    od8[4:4 + 8 * (n + 1)] = torch.from_numpy(offs.view(np.uint8)).cuda()
    with pytest.raises(ecgpu.EcgError) as ei:
        e.ed448_hash_to_curve_ptr(n, dd.data_ptr() + 3, od8.data_ptr() + 4, od.data_ptr(), RO)
    assert ei.value.code == ecgpu.ECG_EINVAL
    e.close()


@pytest.mark.gpu
def test_abi_consttime_and_zeroize_identical(eng):
    import ecgpu

    n = 2051
    msgs = [bytes([i & 0xFF]) * (i % 40) for i in range(n)]

    def run(e):
        return (e.ed448_hash_to_curve(msgs, RO), e.ed448_hash_to_curve(msgs, RO, True), e.ed448_hash_to_scalar(msgs, RO))

    base = run(eng)
    for kw in ({"zeroize": True}, {"consttime": True}, {"zeroize": True, "consttime": True}):
        e = ecgpu.Engine([0], **kw)
        for g, b in zip(run(e), base):
            assert np.array_equal(g, b), kw
        e.close()


@pytest.mark.gpu
def test_abi_timing_brackets_the_hash_kernel():
    import ecgpu

    e = ecgpu.Engine([0])
    e.timing_enable(True)
    e.ed448_hash_to_curve([b"abc"] * 1000, RO)
    e.ed448_hash_to_scalar([b"abc"] * 1000, RO)
    ms, calls = e.timing_read()
    assert calls == 2 and ms > 0
    e.close()


@pytest.mark.gpu
def test_abi_multi_device():
    """two shards (two GPUs when present, else two contexts of device 0): byte-identical to one device"""
    import torch

    import ecgpu

    devs = [0, 1] if torch.cuda.device_count() >= 2 else [0, 0]
    n = 5003
    msgs = [bytes([i & 0xFF]) * (i % 33) for i in range(n)]
    one, two = ecgpu.Engine([0]), ecgpu.Engine(devs)
    for f in (lambda e: e.ed448_hash_to_curve(msgs, bytes(300)), lambda e: e.ed448_hash_to_curve(msgs, RO, True),
              lambda e: e.ed448_hash_to_scalar(msgs, RO)):
        assert np.array_equal(f(one), f(two))
    one.close()
    two.close()
