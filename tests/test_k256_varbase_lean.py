"""The secp256k1 variable-base kernel's policy (FpK256Inline) moves work off the multiplier pipe: beta*x columns in the
window table, 3/2 X^2 by carry chains, and Y3 of the doubling and the mixed addition as one `mul_sub` (two 512-bit
products, one reduction).

 * `mul_sub` / `mul_sub_sqr` on the host twin and the device, against big integers, on boundary operands: weakly
   reduced values in [p, 2^256), all-ones limbs, a*b < c*d, products next to 2^512.
 * The doubling and the mixed addition of the new policy give the same field values as those of the plain inlined
   policy FpK256T<1>, on curve points (checked against the model too), on arbitrary words and in every exceptional branch.
 * Without a GPU: the kernel as group 0 compiles it still fits 128 registers with no more spill than before, and its
   doubling and addition loops issue fewer IMAD.WIDE than the same routine under FpK256T<1>."""
import ctypes
import os
import random
import re
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import pyref
from helpers import random_points

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = os.path.join(ROOT, "tests", "dev")
CSRC = os.path.join(ROOT, "elliptic-curves_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
C = pyref.K256
P = C.p
M256 = (1 << 256) - 1
U32P = ctypes.POINTER(ctypes.c_uint32)


def _words(vals, nw=8):
    out = np.zeros((len(vals), nw), np.uint32)
    for i, v in enumerate(vals):
        for j in range(nw):
            out[i, j] = (v >> (32 * j)) & 0xFFFFFFFF
    return out


def _ints(a):
    return [sum(int(w) << (32 * j) for j, w in enumerate(row)) for row in a]


def _p(a):
    return a.ctypes.data_as(U32P)


class Lib:
    def __init__(self, kind):
        self.lib = L_ = ctypes.CDLL(os.path.join(DEV, "libecgk256leandev.so" if kind == "device" else "libecgk256leandevsim.so"))
        sz = ctypes.c_size_t
        L_.dev_k256l_mul_sub.argtypes = [sz, ctypes.c_int, U32P, U32P, U32P, U32P, U32P]
        L_.dev_k256l_point.argtypes = [sz, ctypes.c_int, ctypes.c_int, U32P, U32P, U32P]
        L_.dev_k256l_error_string.restype = ctypes.c_char_p
        assert L_.dev_k256l_is_device() == (kind == "device")

    def ok(self, err):
        assert err == 0, self.lib.dev_k256l_error_string(err).decode()

    def mul_sub(self, op, a, b, c, d):
        A, B, Cc, D = (_words(v) for v in (a, b, c, d))
        r = np.zeros_like(A)
        self.ok(self.lib.dev_k256l_mul_sub(len(a), op, _p(A), _p(B), _p(Cc), _p(D), _p(r)))
        return _ints(r)

    def point(self, op, lean, jac, aff):
        J = _words([w for X, Y, Z in jac for w in (X, Y, Z)]).reshape(len(jac), 24)
        A = _words([w for x, y in aff for w in (x, y)]).reshape(len(aff), 16)
        out = np.zeros_like(J)
        self.ok(self.lib.dev_k256l_point(len(jac), op, lean, _p(J), _p(A), _p(out)))
        o = _ints(out.reshape(-1, 8))
        return [tuple(o[3 * i:3 * i + 3]) for i in range(len(jac))]


@pytest.fixture(scope="module", params=[pytest.param("host", id="host"), pytest.param("device", id="device", marks=pytest.mark.gpu)])
def lib(request):
    return Lib(request.param)


def _edge_values():
    """weakly reduced and limb-pattern operands: [p, 2^256), all-ones, single limbs, tiny"""
    v = [0, 1, 2, 977, 2**32 + 977, P - 1, P, P + 1, M256 - 1, M256, 2**255, 2**255 - 1, 2**256 - 2**32 - 978]
    v += [((1 << 32) - 1) << (32 * j) for j in range(8)]
    v += [int("0123456789abcdef" * 4, 16), int("fedcba9876543210" * 4, 16), int("ffffffff00000000" * 4, 16)]
    return v


def _mul_sub_cases():
    rng = random.Random(0x1EA5)
    e = _edge_values()
    cases = []
    for a in e:  # products near 2^512 on either side, a*b < c*d, equal products
        cases += [(a, M256, M256, M256), (M256, M256, a, M256), (a, a, a, a), (a, 1, M256, M256), (M256, M256, a, 1), (a, P, P, a)]
    for _ in range(400):
        cases.append(tuple(rng.choice(e) if rng.random() < 0.3 else rng.getrandbits(256) for _ in range(4)))
    for _ in range(200):  # c*d just above / below a*b
        a, b = rng.getrandbits(256), rng.getrandbits(256)
        cases.append((a, b, a, b + rng.choice((-1, 1)) & M256))
    return cases


@pytest.mark.parametrize("op", [0, 1], ids=["ab-cd", "ab-c2"])
def test_mul_sub_matches_big_integers(lib, op):
    cases = _mul_sub_cases()
    a, b, c, d = (list(x) for x in zip(*cases))
    got = lib.mul_sub(op, a, b, c, d)
    for (x, y, z, w), r in zip(cases, got):
        want = (x * y - z * (w if op == 0 else z)) % P
        assert r % P == want and r <= M256, (hex(x), hex(y), hex(z), hex(w))


def _to_aff(J):
    X, Y, Z = (v % P for v in J)
    if Z == 0:
        return None
    zi = pow(Z, -1, P)
    return (X * zi * zi % P, Y * zi * zi * zi % P)


def _jac(A, z, weak=False):
    x, y = A
    X, Y = x * z * z % P, y * z * z * z % P
    if weak:  # the other representative where it fits in 256 bits
        X, Y = (X + P if X + P <= M256 else X), (Y + P if Y + P <= M256 else Y)
    return (X, Y, z)


def _same_field_values(a, b):
    return all((u - v) % P == 0 for u, v in zip(a, b))


def _point_cases():
    rng = random.Random(0xD0B1)
    pts = random_points(C, 48, seed=11)
    jac, aff, model = [], [], []
    for i in range(0, 48, 2):
        A, B = pts[i], pts[i + 1]
        z = rng.randrange(1, P)
        for J, Q in (
            (_jac(A, z), B),                           # generic
            (_jac(A, z), A),                           # P == Q: the doubling branch
            (_jac(A, z), pyref.neg(C, A)),             # P == -Q: the identity
            ((0, 1, 0), B),                            # identity accumulator
            ((0, 1, P), B),                            # identity with Z = p (weakly reduced zero)
            (_jac(A, 1), B),                           # Z = 1
        ):
            jac.append(J)
            aff.append(Q)
    # small x, so that X = x + p (the representative in [p, 2^256)) fits
    for x in range(1, 40):
        A = pyref.lift_x(x)
        if A:
            jac.append(_jac(A, 1, weak=True))
            aff.append(pts[x % 48])
    assert len(jac) > 150
    return jac, aff


@pytest.mark.parametrize("op", [0, 1], ids=["dbl", "madd"])
def test_point_formulas_match_plain_policy_and_model(lib, op):
    jac, aff = _point_cases()
    lean = lib.point(op, 1, jac, aff)
    plain = lib.point(op, 0, jac, aff)
    for J, Q, a, b in zip(jac, aff, lean, plain):
        assert _same_field_values(a, b), (J, Q)
        Pa = _to_aff(J)
        want = pyref.add(C, Pa, Pa) if op == 0 else pyref.add(C, Pa, Q)
        assert _to_aff(a) == want, (J, Q)


@pytest.mark.parametrize("op", [0, 1], ids=["dbl", "madd"])
def test_point_formulas_on_arbitrary_words(lib, op):
    """not curve points: the formulas are polynomial, so both policies must still agree word by word mod p"""
    rng = random.Random(0xA11 + op)
    e = _edge_values()
    pick = lambda: rng.choice(e) if rng.random() < 0.4 else rng.getrandbits(256)  # noqa: E731
    jac = [(pick(), pick(), pick()) for _ in range(600)]
    aff = [(pick(), pick()) for _ in range(600)]
    lean = lib.point(op, 1, jac, aff)
    plain = lib.point(op, 0, jac, aff)
    for J, Q, a, b in zip(jac, aff, lean, plain):
        assert _same_field_values(a, b), (J, Q)


# ---- static checks of the kernel as the library compiles it (no GPU) ----

KERNEL = "_Z19k256_varbase_kernelILi256ELi2EEvPKhS1_S1_mPjS2_S2_m"
PROBE = r"""
#include "ecg_mul.cuh"
using namespace ecg;
// the variable-base routine under the plain inlined policy, in the production kernel's launch bound and phase barriers
__global__ void __launch_bounds__(256, 2) probe_plain(const uint32_t* in, uint32_t* out, uint32_t* gtab) {
  const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  uint32_t k[8];
  Aff P;
  for (int j = 0; j < 8; j++) {
    k[j] = in[j * 65536 + i];
    P.x.v[j] = in[(8 + j) * 65536 + i];
    P.y.v[j] = in[(16 + j) * 65536 + i];
  }
  K256TabRef<FpK256T<1>> tab{gtab + (size_t)blockIdx.x * 256 * 128 + threadIdx.x, 256u};
  Jac r;
  k256_mul_thread<FpK256T<1>, 1>(r, k, P, tab);
  for (int j = 0; j < 8; j++) {
    out[j * 65536 + i] = r.X.v[j];
    out[(8 + j) * 65536 + i] = r.Y.v[j];
    out[(16 + j) * 65536 + i] = r.Z.v[j];
  }
}
"""


def _flags():
    import __graft_entry__ as ge

    return list(ge.NVCC_FLAGS)


def _cubin(src, out, extra):
    cmd = [NVCC] + _flags() + extra + ["-Xptxas", "-v", "-cubin", "-o", out, src]
    r = subprocess.run(cmd, check=True, capture_output=True, text=True, timeout=1800)
    return r.stdout + r.stderr


def _sass(cubin, fn):
    s = subprocess.run([os.path.join(os.path.dirname(NVCC), "cuobjdump"), "-sass", "-fun", fn, cubin], check=True,
                       capture_output=True, text=True).stdout
    ins = []
    for line in s.splitlines():
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*)", line)
        if m:
            ins.append((int(m.group(1), 16), m.group(2)))
    return ins


def loop_imad_wide(ins):
    """IMAD.WIDE in the doubling loop and in the addition loop: the loops that branch back to the instruction after
    the first and the second BAR.SYNC of the window loop"""
    bars = [a for a, t in ins if "BAR.SYNC" in t]
    assert len(bars) == 2, bars
    step = ins[1][0] - ins[0][0]
    counts = []
    for b in bars:
        back = [a for a, t in ins if (m := re.search(r"\bBRA\b.*?(0x[0-9a-f]+)", t)) and int(m.group(1), 16) == b + step and a > b]
        assert len(back) == 1, (hex(b), back)
        counts.append(sum("IMAD.WIDE" in t for a, t in ins if b + step <= a <= back[0]))
    return counts


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    d = tmp_path_factory.mktemp("lean_sass")
    probe_src = d / "probe.cu"
    probe_src.write_text(PROBE)
    jobs = [(os.path.join(CSRC, "ecgpu.cu"), str(d / "tu0.cubin"), ["-DECG_TU=0"]),
            (str(probe_src), str(d / "probe.cubin"), [f"-I{CSRC}"])]
    with ThreadPoolExecutor(2) as ex:
        logs = list(ex.map(lambda j: _cubin(*j), jobs))
    return d, logs[0]


def test_kernel_registers_and_spills(compiled):
    _, log = compiled
    m = re.search(re.escape(KERNEL) + r"' for 'sm_90a'\s+ptxas info\s+: Function properties for \S+\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\s+ptxas info\s+: Used (\d+) registers", log)
    assert m, log[-2000:]
    stack, st, ld, regs = map(int, m.groups())
    # the plain inlined body (FpK256T<1>) compiled to 128 registers, 80 B spill stores, 96 B spill loads
    assert regs <= 128 and st <= 80 and ld <= 96, (regs, st, ld)


def test_loops_issue_fewer_imad_wide(compiled):
    d, _ = compiled
    new_dbl, new_add = loop_imad_wide(_sass(str(d / "tu0.cubin"), KERNEL))
    old_dbl, old_add = loop_imad_wide(_sass(str(d / "probe.cubin"), "_Z11probe_plainPKjPjS1_"))
    # doubling: mul_small(3) (8) and one reduction (8 + 1); addition: beta*x (64 + 9) and one reduction (8 + 1)
    assert new_dbl <= old_dbl - 8, (new_dbl, old_dbl)
    assert new_add <= old_add - 40, (new_add, old_add)
