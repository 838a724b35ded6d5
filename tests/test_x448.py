"""X448 (RFC 7748): the Python model, the Curve448 field, the ladder step and the per-pair routine as the kernel compiles
them, and ecg_x448_batch through the C ABI, the Python mirror and the C++ mirror.

Oracles: the reference's own vectors (tests/golden/x448.json: RFC 7748 sections 5.2 and 6.2 and the low-order encodings),
OpenSSL's X448 through `cryptography`, and the model in x448_model.py (Python integers).  The device library
(tests/dev/x448_dev.cu, both field variants under x448_kernel's launch bound) runs under the `gpu` marker; its host twin
(the same bodies over the C emulation of the carry primitives) runs everywhere, and the device must give its bits."""
import ctypes
import json
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

import x448_model as M

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = os.path.join(HERE, "dev")
LIB = os.path.join(ROOT, "elliptic-curves_b200", "libecgpu.so")
GOLDEN = json.load(open(os.path.join(HERE, "golden", "x448.json")))
U32P = ctypes.POINTER(ctypes.c_uint32)
U8P = ctypes.POINTER(ctypes.c_uint8)
P, W = M.P, 1 << 448
OPS = {"add": 0, "sub": 1, "mul": 2, "sqr": 3, "neg": 4, "mul_small": 5, "inv": 6, "normalize": 7, "cswap1": 8, "cswap0": 9}
VARIANTS = (0, 1)  # 0: every field operation inlined, 1: mul / sqr as device functions
EDGES = [0, 1, 2, P - 2, P - 1, P, P + 1, 2**224 - 1, 2**224, 2**224 + 1, W - 2**224, W - 1]


def _b(h):
    return bytes.fromhex(h)


def openssl_x448(k: bytes, u: bytes):
    """OpenSSL's X448; None where it refuses an all-zero result"""
    from cryptography.hazmat.primitives.asymmetric.x448 import X448PrivateKey, X448PublicKey

    try:
        return X448PrivateKey.from_private_bytes(k).exchange(X448PublicKey.from_public_bytes(u))
    except ValueError:
        return None


def special_u():
    return [bytes.fromhex(h) for h in GOLDEN["low_order"].values()] + [
        v.to_bytes(56, "little") for v in (P, P + 1, W - 1, 5, P + 5, W - 2**224)]


def random_pairs(n, seed):
    """uniform scalars and u values (about half of them on the twist), with every 8th u in [p, 2^448)"""
    rng = random.Random(seed)
    ks = [rng.getrandbits(448).to_bytes(56, "little") for _ in range(n)]
    us = [(P + rng.getrandbits(224) if i % 8 == 3 else rng.getrandbits(448)).to_bytes(56, "little") for i in range(n)]
    return ks, us


# ---- the model ----------------------------------------------------------------------------------------------------------
def test_model_reproduces_golden_vectors():
    for v in GOLDEN["fixed"]:
        assert M.x448(_b(v["k"]), _b(v["u"])).hex() == v["out"]
    ab = GOLDEN["alice_bob"]
    assert M.x448(_b(ab["alice_priv"]), M.GENERATOR).hex() == ab["alice_pub"]
    assert M.x448(_b(ab["bob_priv"]), M.GENERATOR).hex() == ab["bob_pub"]
    assert M.x448(_b(ab["alice_priv"]), _b(ab["bob_pub"])).hex() == ab["shared"]
    assert M.x448(_b(ab["bob_priv"]), _b(ab["alice_pub"])).hex() == ab["shared"]
    k = u = M.GENERATOR
    for i in range(1000):
        k, u = M.x448(k, u), k
        if i == 0:
            assert k.hex() == GOLDEN["iterations"]["1"]
    assert k.hex() == GOLDEN["iterations"]["1000"]
    assert sorted(GOLDEN["low_order"].values()) == sorted(b.hex() for b in M.LOW_ORDER)


def test_model_against_openssl():
    ks, us = random_pairs(1024 - 9, seed=448)
    ks += [bytes(56), b"\xff" * 56, ks[0]] + ks[:6]
    us += special_u()[:3] + [us[1]] + special_u()[3:]
    refused = 0
    for k, u in zip(ks, us):
        o = openssl_x448(k, u)
        if o is None:  # OpenSSL refuses an all-zero result; the reference (and the model) return it
            refused += 1
            assert M.x448(k, u) == bytes(56)
        else:
            assert M.x448(k, u) == o, (k.hex(), u.hex())
    assert refused >= 3  # the low-order u values
    assert [M.u_ok(u) for u in special_u()] == [False, False, False] + [True] * 6


# ---- device library and its host twin -----------------------------------------------------------------------------------
class X448Dev:
    def __init__(self, kind):
        import __graft_entry__ as ge

        ge.build()
        self.kind = kind
        L = self.lib = ctypes.CDLL(os.path.join(DEV, "libecgx448dev.so" if kind == "device" else "libecgx448devsim.so"))
        L.dev_x448_fe_op.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_size_t, U32P, U32P, U32P, U32P]
        L.dev_x448_step.argtypes = [ctypes.c_int, ctypes.c_size_t, U32P, U32P]
        L.dev_x448_one.argtypes = [ctypes.c_int, ctypes.c_size_t, U8P, U8P, U8P, U8P]
        L.dev_x448_error_string.restype = ctypes.c_char_p
        assert L.dev_x448_is_device() == (1 if kind == "device" else 0)

    def ok(self, rc):
        assert rc == 0, f"rc {rc}: {self.lib.dev_x448_error_string(rc).decode()}"

    @staticmethod
    def pack(vals):
        return np.frombuffer(b"".join(v.to_bytes(56, "little") for v in vals), np.uint32).copy()

    @staticmethod
    def unpack(arr):
        b = np.ascontiguousarray(arr).view(np.uint8).reshape(-1, 56)
        return [int.from_bytes(r.tobytes(), "little") for r in b]

    def fe_op(self, v, op, a, b):
        n = len(a)
        A, B = self.pack(a), self.pack(b)
        raw, norm = np.zeros(14 * n, np.uint32), np.zeros(14 * n, np.uint32)
        self.ok(self.lib.dev_x448_fe_op(v, OPS[op], n, _p(A), _p(B), _p(raw), _p(norm)))
        return raw, norm

    def step(self, v, states):
        n = len(states)
        inp = self.pack([x for s in states for x in s])
        out = np.zeros(56 * n, np.uint32)
        self.ok(self.lib.dev_x448_step(v, n, _p(inp), _p(out)))
        return out

    def one(self, v, ks, us):
        n = len(ks)
        K = np.frombuffer(b"".join(ks), np.uint8).copy()
        U = np.frombuffer(b"".join(us), np.uint8).copy() if us is not None else None
        out, ok = np.zeros(56 * n, np.uint8), np.zeros(n, np.uint8)
        self.ok(self.lib.dev_x448_one(v, n, _p(K, U8P), _p(U, U8P) if U is not None else None, _p(out, U8P), _p(ok, U8P)))
        return [out[56 * i:56 * i + 56].tobytes() for i in range(n)], ok


def _p(a, t=U32P):
    return a.ctypes.data_as(t)


_BACKENDS = {}


def backend(kind):
    if kind not in _BACKENDS:
        _BACKENDS[kind] = X448Dev(kind)
    return _BACKENDS[kind]


@pytest.fixture(scope="module", params=[pytest.param("host", id="host"), pytest.param("device", id="device", marks=pytest.mark.gpu)])
def be(request):
    return backend(request.param)


def field_inputs(n, seed):
    """every ordered pair of edge values, then limb patterns and uniform values in [0, 2^448)"""
    rng = random.Random(seed)
    pairs = [(x, y) for x in EDGES for y in EDGES]
    limbs = [0, 1, 0xFFFFFFFF, 0xFFFFFFFE]
    pats = [sum((rng.choice(limbs) if rng.random() < 0.8 else rng.getrandbits(32)) << (32 * i) for i in range(14)) for _ in range(512)]
    uni = [rng.getrandbits(448) for _ in range(n)]
    a = [x for x, _ in pairs] + pats + uni
    b = [y for _, y in pairs] + pats[::-1] + [rng.getrandbits(448) for _ in range(n)]
    return a, b


def expect(op, x, y):
    return {"add": x + y, "sub": x - y, "mul": x * y, "sqr": x * x, "neg": -x, "mul_small": M.A24 * x,
            "inv": pow(x, P - 2, P), "normalize": x}[op] % P


@pytest.mark.parametrize("v", VARIANTS)
@pytest.mark.parametrize("op", list(OPS))
def test_field_ops(be, v, op):
    """congruence and the documented range of the raw result (below 2^448; below p for normalize), and a canonical
    normalised form; cswap exchanges the raw limbs exactly.  The device gives the host twin's bits."""
    a, b = field_inputs(4096, seed=OPS[op])
    raw, norm = be.fe_op(v, op, a, b)
    R, N = be.unpack(raw), be.unpack(norm)
    for i, (x, y) in enumerate(zip(a, b)):
        if op == "cswap1":
            assert R[i] == y
            continue
        if op == "cswap0":
            assert R[i] == x
            continue
        e = expect(op, x, y)
        assert R[i] < W and R[i] % P == e, (op, hex(x), hex(y))
        assert N[i] == e
        if op == "normalize":
            assert R[i] < P
    if be.kind == "device":
        hraw, hnorm = backend("host").fe_op(v, op, a, b)
        assert np.array_equal(raw, hraw) and np.array_equal(norm, hnorm)


def step_states(n, seed):
    """random projective states, the identity (W = 0) in either slot, and edge values as coordinates"""
    rng = random.Random(seed)
    st = []
    for i in range(n):
        s = [rng.getrandbits(448) for _ in range(5)]
        if i % 7 == 0:
            s[1] = 0 if i % 14 == 0 else P  # (x2 : z2) = identity, W = 0 as 0 or as p
        if i % 11 == 0:
            s[3] = 0
        st.append(s)
    st += [[EDGES[i % 12], EDGES[(i // 12) % 12], EDGES[(i * 5) % 12], EDGES[(i * 7 + 1) % 12], EDGES[(i * 3 + 2) % 12]] for i in range(144)]
    return st


@pytest.mark.parametrize("v", VARIANTS)
def test_ladder_step(be, v):
    st = step_states(1024, seed=7)
    out = be.unpack(be.step(v, st))
    for i, s in enumerate(st):
        got = out[4 * i:4 * i + 4]
        assert all(g < W for g in got)
        assert [g % P for g in got] == list(M.ladder_step(*[x % P for x in s])), i
    if be.kind == "device":
        assert np.array_equal(be.step(v, st), backend("host").step(v, st))


def one_cases(n_random):
    ks, us = [], []
    for vec in GOLDEN["fixed"]:
        ks.append(_b(vec["k"]))
        us.append(_b(vec["u"]))
    ab = GOLDEN["alice_bob"]
    ks += [_b(ab["alice_priv"]), _b(ab["bob_priv"]), _b(ab["alice_priv"]), _b(ab["bob_priv"])]
    us += [M.GENERATOR, M.GENERATOR, _b(ab["bob_pub"]), _b(ab["alice_pub"])]
    for k in (bytes(56), b"\xff" * 56, _b(ab["alice_priv"])):
        for u in special_u():
            ks.append(k)
            us.append(u)
    rk, ru = random_pairs(n_random, seed=5)
    return ks + rk, us + ru


@pytest.mark.parametrize("v", VARIANTS)
def test_x448_one(be, v):
    ks, us = one_cases(512)
    out, ok = be.one(v, ks, us)
    for i, (k, u) in enumerate(zip(ks, us)):
        assert out[i] == M.x448(k, u), i
        assert ok[i] == M.u_ok(u)
    g, gok = be.one(v, ks[:8], None)  # u = NULL: the generator
    assert g == [M.x448(k, M.GENERATOR) for k in ks[:8]] and list(gok) == [1] * 8
    if be.kind == "device":
        assert out == backend("host").one(v, ks, us)[0]


@pytest.mark.parametrize("v", VARIANTS)
def test_x448_one_iterations(be, v):
    k = u = M.GENERATOR
    for i in range(1000):
        out, _ = be.one(v, [k], [u])
        k, u = out[0], k
        if i == 0:
            assert k.hex() == GOLDEN["iterations"]["1"]
    assert k.hex() == GOLDEN["iterations"]["1000"]


# ---- the C ABI, the Python and C++ mirrors ------------------------------------------------------------------------------
def test_abi_null_ctx():
    import ecgpu

    lib = ecgpu.load_library()
    k = np.zeros(56, np.uint8)
    out = np.zeros(56, np.uint8)
    assert lib.ecg_x448_batch(None, 1, k.ctypes.data, None, out.ctypes.data, None) == ecgpu.ECG_EINVAL
    assert lib.ecg_x448_batch(None, 0, None, None, None, None) == ecgpu.ECG_EINVAL


CPP = r"""
#include "ecgpu.hpp"
#include <cstdio>
int main() {
  try {
    ecgpu::Engine eng(ECG_SECP256K1);
    std::vector<ecgpu::Engine::X448Bytes> k(2), u(2);
    const char* hk[2] = {"%(k0)s", "%(k1)s"};
    const char* hu[2] = {"%(u0)s", "%(u1)s"};
    for (int j = 0; j < 2; j++)
      for (int i = 0; i < 56; i++) {
        unsigned b;
        std::sscanf(hk[j] + 2 * i, "%%2x", &b); k[j][i] = (uint8_t)b;
        std::sscanf(hu[j] + 2 * i, "%%2x", &b); u[j][i] = (uint8_t)b;
      }
    std::vector<bool> ok;
    auto r = eng.x448(k, u, &ok);
    auto pub = eng.x448(k);
    char hex[113];
    for (int i = 0; i < 56; i++) std::snprintf(hex + 2 * i, 3, "%%02x", r[0][i]);
    std::printf("out0=%%s\n", hex);
    for (int i = 0; i < 56; i++) std::snprintf(hex + 2 * i, 3, "%%02x", pub[1][i]);
    std::printf("pub1=%%s ok=%%d%%d\n", hex, (int)ok[0], (int)ok[1]);
    return 0;
  } catch (const ecgpu::Error& e) {
    std::printf("error %%d\n", (int)e.code);
    return e.code == ECG_ECUDA ? 42 : 3;  // 42: no GPU -> a loud failure, no CPU fallback
  }
}
"""


def _cpp_run():
    ab = GOLDEN["alice_bob"]
    src_text = CPP % {"k0": GOLDEN["fixed"][0]["k"], "u0": GOLDEN["fixed"][0]["u"], "k1": ab["bob_priv"], "u1": GOLDEN["low_order"]["LOW_B"]}
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "x.cpp"), os.path.join(d, "x")
        open(src, "w").write(src_text)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "elliptic-curves_b200", "host"), src, LIB,
                               "-Wl,-rpath," + os.path.dirname(LIB), "-o", exe])
        p = subprocess.run([exe], capture_output=True, text=True, timeout=300)
        return p.returncode, p.stdout + p.stderr


def test_cpp_mirror_x448_compiles_and_links():
    import torch

    rc, out = _cpp_run()
    if torch.cuda.is_available():
        assert rc == 0, out
    else:
        assert rc == 42, out  # ECG_ECUDA without a GPU


@pytest.mark.gpu
def test_cpp_mirror_x448_for_real():
    rc, out = _cpp_run()
    assert rc == 0, out
    assert f"out0={GOLDEN['fixed'][0]['out']}" in out
    assert f"pub1={GOLDEN['alice_bob']['bob_pub']} ok=10" in out


@pytest.fixture(scope="module")
def eng():
    import ecgpu

    e = ecgpu.Engine([0])
    yield e
    e.close()


def _arr(recs):
    return np.frombuffer(b"".join(recs), np.uint8).copy()


@pytest.mark.gpu
def test_abi_golden(eng):
    for vec in GOLDEN["fixed"]:
        out, ok = eng.x448(_arr([_b(vec["k"])]), _arr([_b(vec["u"])]))
        assert out[0].tobytes().hex() == vec["out"] and ok[0] == 1
    ab = GOLDEN["alice_bob"]
    pubs, _ = eng.x448(_arr([_b(ab["alice_priv"]), _b(ab["bob_priv"])]))
    assert [r.tobytes().hex() for r in pubs] == [ab["alice_pub"], ab["bob_pub"]]
    shared, ok = eng.x448(_arr([_b(ab["alice_priv"]), _b(ab["bob_priv"])]), _arr([_b(ab["bob_pub"]), _b(ab["alice_pub"])]))
    assert [r.tobytes().hex() for r in shared] == [ab["shared"]] * 2 and list(ok) == [1, 1]
    ks, _ = random_pairs(300, seed=11)
    g_none, _ = eng.x448(_arr(ks))
    g_five, _ = eng.x448(_arr(ks), _arr([M.GENERATOR] * 300))
    assert np.array_equal(g_none, g_five)


@pytest.mark.gpu
def test_abi_iterations(eng):
    k = u = M.GENERATOR
    for i in range(1000):
        out, _ = eng.x448(_arr([k]), _arr([u]))
        k, u = out[0].tobytes(), k
        if i == 0:
            assert k.hex() == GOLDEN["iterations"]["1"]
    assert k.hex() == GOLDEN["iterations"]["1000"]


@pytest.mark.gpu
def test_abi_against_openssl(eng):
    n = 1 << 16
    ks, us = random_pairs(n, seed=65536)
    out, ok = eng.x448(_arr(ks), _arr(us))
    assert ok.all()
    for i in range(n):
        o = openssl_x448(ks[i], us[i])
        assert out[i].tobytes() == (o if o is not None else M.x448(ks[i], us[i])), i


@pytest.mark.gpu
def test_abi_low_order_flags(eng):
    us = special_u()
    ks, _ = random_pairs(len(us), seed=3)
    out, ok = eng.x448(_arr(ks), _arr(us))
    assert list(ok) == [0, 0, 0] + [1] * (len(us) - 3)
    for i in range(len(us)):
        assert out[i].tobytes() == M.x448(ks[i], us[i])
    assert out[3].tobytes() == bytes(56)  # u = p: a non-canonical encoding of 0, not refused, the identity


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 257, (1 << 18) + 3])
def test_abi_ragged_sizes(eng, n):
    ks, us = random_pairs(n, seed=n)
    out, ok = eng.x448(_arr(ks), _arr(us)) if n else eng.x448(np.zeros(0, np.uint8), np.zeros(0, np.uint8))
    assert out.shape == (n, 56) and ok.shape == (n,)
    for i in range(n):
        assert out[i].tobytes() == openssl_x448(ks[i], us[i]), i


@pytest.mark.gpu
def test_abi_device_pointers():
    import torch

    import ecgpu

    n = 4099
    ks, us = random_pairs(n, seed=99)
    ref, _ = ecgpu.Engine([0]).x448(_arr(ks), _arr(us))
    e = ecgpu.Engine([0], device_ptrs=True)
    kd, ud = torch.from_numpy(_arr(ks)).cuda(), torch.from_numpy(_arr(us)).cuda()
    od, okd = torch.zeros(56 * n, dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.uint8, device="cuda")
    launches = e.kernel_launches
    e.x448_ptr(n, kd.data_ptr(), ud.data_ptr(), od.data_ptr(), okd.data_ptr())
    torch.cuda.synchronize()
    assert e.kernel_launches == launches + 1
    assert np.array_equal(od.cpu().numpy().reshape(n, 56), ref) and bool((okd == 1).all())
    e.x448_ptr(n, kd.data_ptr(), 0, od.data_ptr(), 0)  # u = generator, no flags
    torch.cuda.synchronize()
    g, _ = ecgpu.Engine([0]).x448(_arr(ks))
    assert np.array_equal(od.cpu().numpy().reshape(n, 56), g)
    e.close()


@pytest.mark.gpu
def test_abi_zeroize_and_consttime_flags(eng):
    import ecgpu

    n = 2051
    ks, us = random_pairs(n, seed=2051)
    ref, rok = eng.x448(_arr(ks), _arr(us))
    for kw in ({"zeroize": True}, {"consttime": True}, {"zeroize": True, "consttime": True}):
        e = ecgpu.Engine([0], **kw)
        out, ok = e.x448(_arr(ks), _arr(us))
        assert np.array_equal(out, ref) and np.array_equal(ok, rok), kw
        e.close()


@pytest.mark.gpu
def test_abi_timing_brackets_the_ladder(eng):
    n = 4096
    ks, us = random_pairs(n, seed=4)
    eng.timing_enable(True)
    eng.x448(_arr(ks), _arr(us))
    ms, calls = eng.timing_read()
    eng.timing_enable(False)
    assert calls == 1 and ms > 0


@pytest.mark.gpu
def test_abi_multi_device():
    import torch

    import ecgpu

    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    n = 5003
    ks, us = random_pairs(n, seed=2)
    ref, _ = ecgpu.Engine([0]).x448(_arr(ks), _arr(us))
    e = ecgpu.Engine([0, 1])
    out, _ = e.x448(_arr(ks), _arr(us))
    assert np.array_equal(out, ref)
    e.close()
