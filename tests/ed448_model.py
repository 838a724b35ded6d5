"""Ed448 (RFC 8032) in Python integers: the model the Ed448 tests check the device, its host twin and OpenSSL against.

verify() restates the reference's VerifyingKey::from_bytes + verify_inner (ed448-goldilocks/src/sign/verifying_key.rs)
with its decoders, quirks included:
  - S: byte 56 must be 0, the other 56 bytes little-endian below ell, and S != 0;
  - A and R (CompressedEdwardsY::decompress, edwards/affine.rs): y = bytes 0..55 little-endian reduced mod p (y >= p is
    accepted), the sign of x is bit 7 of byte 56 and bits 0-6 of byte 56 are ignored; refused when (1 - y^2) / (1 - d y^2)
    is not a square or the point is not in the prime-order subgroup; then refused if it is the identity;
  - k = SHAKE256(dom4 || R bytes || A bytes || M, 114) mod ell over the bytes as given, and [S]B == R + [k]A.
The subgroup test here is the definition, [ell]P == O; the device uses a cheaper predicate (torsion_free_fast) that the
tests compare with this one.

sign() is RFC 8032 signing, used only to make test signatures (contexts, Ed448ph, non-canonical encodings of A and R)."""
import hashlib

P = 2**448 - 2**224 - 1
D = P - 39081
L = 2**446 - 13818066809895115352007386748515426880336692474882178609894547503885
IDENTITY = (0, 1)
# the torsion points besides the identity: (0, -1) of order 2, (+-1, 0) of order 4
TORSION = ((0, P - 1), (1, 0), (P - 1, 0))


def inv(a):
    return pow(a, P - 2, P)


def add(p1, p2):
    (x1, y1), (x2, y2) = p1, p2
    t = D * x1 * x2 * y1 * y2 % P
    return (x1 * y2 + y1 * x2) * inv(1 + t) % P, (y1 * y2 - x1 * x2) * inv(1 - t) % P


def neg(pt):
    return (-pt[0]) % P, pt[1]


def _padd(p1, p2):
    """complete addition in projective coordinates (X : Y : Z), a = 1 (no inversion)"""
    (x1, y1, z1), (x2, y2, z2) = p1, p2
    a, b = z1 * z2 % P, x1 * x2 % P
    c, dd = y1 * y2 % P, D * (x1 * x2 % P) * (y1 * y2 % P) % P
    bb = a * a % P
    e, f = (bb - dd) % P, (bb + dd) % P
    return (a * e * ((x1 + y1) * (x2 + y2) - b - c) % P, a * f * (c - b) % P, e * f % P)


def mul(k, pt):
    """[k] pt (double and add over projective coordinates, one inversion at the end)"""
    r, q = (0, 1, 1), (pt[0], pt[1], 1)
    while k:
        if k & 1:
            r = _padd(r, q)
        q = _padd(q, q)
        k >>= 1
    zi = inv(r[2])
    return r[0] * zi % P, r[1] * zi % P


def sqrt(a):
    r = pow(a % P, (P + 1) // 4, P)
    return r if r * r % P == a % P else None


def is_square(a):
    return pow(a % P, (P - 1) // 2, P) != P - 1


def on_curve(pt):
    x, y = pt
    return (x * x + y * y - 1 - D * x * x * y * y) % P == 0


def encode(pt):
    x, y = pt
    return (y | (x & 1) << 455).to_bytes(57, "little")


def decompress_unchecked(b: bytes):
    """x and y of the encoding, or None when (1 - y^2) / (1 - d y^2) has no square root (decompress_unchecked)"""
    assert len(b) == 57
    y = int.from_bytes(b[:56], "little") % P
    u, v = (1 - y * y) % P, (1 - D * y * y) % P
    x = sqrt(u * inv(v))
    if x is None:
        return None
    if (x & 1) != (b[56] >> 7):
        x = (-x) % P
    return x, y


def torsion_free(pt):
    return mul(L, pt) == IDENTITY


def torsion_free_fast(y):
    """the device's predicate on y alone (P and -P share it): y^2 = 1 is the identity (torsion free) or (0, -1) (not);
    otherwise P lies in 2E iff (1 - d)(1 - d y^2) is a square, and a half Q = (x1, y1) of P, t = y1^2, lies in 2E iff
    t (1 - d t) is not a square, for either root of the quadratic that t solves"""
    y %= P
    if (y * y - 1) % P == 0:
        return y == 1
    n = (1 - D * y * y) % P
    r = sqrt((1 - D) * n)
    if r is None:
        return False
    den = D * (1 - y * y) % P
    num = ((n + r) * (1 - y) + y * den) % P
    return not is_square(num * (den - D * num)) and num * (den - D * num) % P != 0


def decompress(b: bytes):
    """CompressedEdwardsY::decompress: None unless the encoding decodes to a point of the prime-order subgroup"""
    pt = decompress_unchecked(b)
    if pt is None or not on_curve(pt) or not torsion_free(pt):
        return None
    return pt


def shake256(data: bytes, n=114) -> bytes:
    return hashlib.shake_256(data).digest(n)


def dom4(phflag: int, ctx: bytes) -> bytes:
    assert len(ctx) <= 255
    return b"SigEd448" + bytes([phflag, len(ctx)]) + ctx


def scalar_wide(b: bytes) -> int:
    """EdwardsScalar::from_bytes_mod_order_wide: 114 bytes little-endian mod ell"""
    return int.from_bytes(b, "little") % L


def s_ok(s57: bytes) -> bool:
    """byte 56 zero, S < ell, S != 0 (verify_inner's checks and EdwardsScalar::from_canonical_bytes)"""
    s = int.from_bytes(s57[:56], "little")
    return s57[56] == 0 and 0 < s < L


B_BYTES = bytes.fromhex(
    "14fa30f25b790898adc8d74e2c13bdfdc4397ce61cffd33ad7c2a0051e9c78874098a36c7373ea4b62c7c9563720768824bcb66e71463f6900")
B = decompress_unchecked(B_BYTES)


def verify(pk: bytes, sig: bytes, msg: bytes, ctx: bytes = b"", prehashed: bool = False) -> bool:
    """VerifyingKey::from_bytes(pk) followed by verify_inner(sig, phflag, ctx, msg); msg is PH(M) when prehashed"""
    assert len(pk) == 57 and len(sig) == 114
    A = decompress(pk)
    if A is None or A == IDENTITY:
        return False
    r_bytes, s_bytes = sig[:57], sig[57:]
    if s_bytes[56] != 0:
        return False
    s = int.from_bytes(s_bytes[:56], "little")
    if s >= L:
        return False
    R = decompress(r_bytes)
    if R is None or R == IDENTITY or s == 0:
        return False
    k = scalar_wide(shake256(dom4(1 if prehashed else 0, ctx) + r_bytes + pk + msg))
    return mul(s, B) == add(R, mul(k, A))


def expand_secret(seed: bytes):
    h = shake256(seed, 114)
    a = bytearray(h[:57])
    a[0] &= 0xFC
    a[56] = 0
    a[55] |= 0x80
    return int.from_bytes(a, "little"), h[57:]


def public_key(seed: bytes) -> bytes:
    return encode(mul(expand_secret(seed)[0], B))


def sign(seed: bytes, msg: bytes, ctx: bytes = b"", prehashed: bool = False, pk: bytes = None, r_bytes_of=None) -> bytes:
    """RFC 8032 section 5.2.6 signing (msg is PH(M) when prehashed).  pk: the public-key bytes to hash (default: the
    canonical encoding); r_bytes_of: a function giving the R bytes to hash and emit from the canonical ones (test
    signatures with non-canonical encodings, which the reference accepts)"""
    a, prefix = expand_secret(seed)
    if pk is None:
        pk = encode(mul(a, B))
    dom = dom4(1 if prehashed else 0, ctx)
    r = scalar_wide(shake256(dom + prefix + msg))
    rb = encode(mul(r, B))
    if r_bytes_of is not None:
        rb = r_bytes_of(rb)
    k = scalar_wide(shake256(dom + rb + pk + msg))
    return rb + ((r + k * a) % L).to_bytes(57, "little")


def prehash(msg: bytes) -> bytes:
    """PH(M) of Ed448ph: SHAKE256(M, 64)"""
    return shake256(msg, 64)
