"""Decaf448 (RFC 9496) in Python integers: the model the Decaf448 tests check the device, its host twin and the C ABI
against.  Two restatements live here side by side.

The reference's own (ed448-goldilocks/src/decaf/points.rs, field/element.rs), on the twisted curve -x^2 + y^2 =
1 + TWISTED_D x^2 y^2 (a = -1, TWISTED_D = -39082), in its extended coordinates (X : Y : Z : T):
  - tw_decompress: CompressedDecaf::decompress (points.rs:555-593): s canonical (< p), s even, the inverse square root
    exists, the point is on the curve;
  - tw_compress: DecafPoint::compress (points.rs:49-67);
  - tw_add: ExtendedPoint::add_extended (curve/twedwards/extended.rs:82-98) followed by to_extended (T = T1 T2);
  - tw_map: FieldElement::map_to_curve_decaf448 (field/element.rs:466-507).

The device's, on the untwisted Edwards448 curve x^2 + y^2 = 1 + d x^2 y^2 (d = -39081) of ed448_model, RFC 9496's
decaf448 formulas (decode / encode): a representative there carries 2-torsion only, and encode is invariant under
adding (0, -1), so the Ed448 variable-base and fixed-base routines serve Decaf448 unchanged.  G0 = decode(GENERATOR)
equals [-2]B modulo the 2-torsion, where B is the Ed448 base point: [k]G = encode([-2k mod ell] B).

Hash to group and hash to scalar follow hash2curve with ExpandMsgXof<Shake256> at security level 28
(lib.rs:159-164, hash2curve/src/group_digest.rs, hash2field/expand_msg/xof.rs)."""
import hashlib

import ed448_model as M

P, L = M.P, M.L
D = M.D  # untwisted d = -39081
TW_D = P - 39082  # twisted d
NEG_D = 39081
DECAF_FACTOR = 0x22D962FBEB24F7683BF68D722FA26AA0A1F1A7B8A5B8D54B64A2D780968C14BA839A66F4FD6EDED260337BF6AA20CE529642EF0F45572736
SQRT_MINUS_D = pow(NEG_D, (P + 1) // 4, P)  # sqrt(-d), as the appendix of RFC 9496 section 5 writes it
INV_SQRT_MINUS_D = pow(SQRT_MINUS_D, P - 2, P)
ONE_MINUS_TWO_D = 78163  # 1 - 2 d_untwisted
IDENTITY_BYTES = bytes(56)
GENERATOR_BYTES = bytes([0x66] * 28 + [0x33] * 28)
HASH_TO_CURVE_ID = b"decaf448_XOF:SHAKE256_D448MAP_RO_"
ENCODE_TO_CURVE_ID = b"decaf448_XOF:SHAKE256_D448MAP_NU_"


def isr(a):
    """FieldElement::inverse_square_root: a^((p - 3) / 4) and whether a is a non-zero square"""
    r = pow(a % P, (P - 3) // 4, P)
    return r, r * r * a % P == 1


def neg_(v):
    """v % 2 == 1 is 'negative' (FieldElement::is_negative)"""
    return (v % P) & 1


def absv(v):
    v %= P
    return (P - v) % P if v & 1 else v


# ---- the reference's twisted restatement ---------------------------------------------------------------------------------
def tw_on_curve(pt):
    X, Y, Z, T = pt
    return (X * Y - Z * T) % P == 0 and (Y * Y - X * X - Z * Z - TW_D * T * T) % P == 0


def tw_decompress(b: bytes):
    """CompressedDecaf::decompress: (X, Y, Z, T) or None"""
    assert len(b) == 56
    s = int.from_bytes(b, "little") % P
    canonical = s.to_bytes(56, "little") == b
    ss = s * s % P
    u1, u2 = (1 - ss) % P, (1 + ss) % P
    u1_sqr = u1 * u1 % P
    v = (ss * (4 * 39082) + u1_sqr) % P  # NEG_FOUR_TIMES_TWISTED_D = 156328
    I, ok = isr(v * u1_sqr)
    Dx = I * u1 % P
    Dxs = 2 * s * Dx % P
    X = Dxs * I * v % P
    if neg_(Dxs * DECAF_FACTOR):
        X = (-X) % P
    Y = Dx * u2 % P
    pt = (X, Y, 1, X * Y % P)
    if ok and tw_on_curve(pt) and canonical and not (s & 1):
        return pt
    return None


def tw_compress(pt) -> bytes:
    X, _, Z, T = pt
    xx_tt = (X + T) * (X - T) % P
    r, _ = isr(X * X * xx_tt * NEG_D)
    ratio = r * xx_tt % P
    if neg_(ratio * DECAF_FACTOR):
        ratio = (-ratio) % P
    k = (ratio * Z - T) % P
    s = absv(k * NEG_D * r * X)
    return s.to_bytes(56, "little")


def tw_add(p1, p2):
    X1, Y1, Z1, T1 = p1
    X2, Y2, Z2, T2 = p2
    A, B = X1 * X2 % P, Y1 * Y2 % P
    C, Dd = T1 * T2 * TW_D % P, Z1 * Z2 % P
    E = ((X1 + Y1) * (X2 + Y2) - A - B) % P
    F, G, H = (Dd - C) % P, (Dd + C) % P, (B + A) % P
    return E * F % P, G * H % P, F * G % P, E * H % P


TW_IDENTITY = (0, 1, 1, 0)


def tw_mul(k, pt):
    acc, q = TW_IDENTITY, pt
    while k:
        if k & 1:
            acc = tw_add(acc, q)
        q = tw_add(q, q)
        k >>= 1
    return acc


def tw_map(u):
    """FieldElement::map_to_curve_decaf448 (twisted extended output)"""
    u %= P
    r = (-u * u) % P
    a = (r - 1) % P
    b = a * D % P
    a = (b + 1) % P
    b = (b - r) % P
    c = a * b % P
    n = (r + 1) * ONE_MINUS_TWO_D % P
    a = c * n % P
    bb, square = isr(a)
    c = 1 if square else u
    e = bb * c % P
    a = n * e % P
    if (not neg_(a)) ^ square:
        a = (-a) % P
    c = e * ONE_MINUS_TWO_D % P
    b = c * c % P
    e = (r - 1) % P
    c = b * e % P
    b = c * n % P
    if square:
        b = (-b) % P
    b = (b - 1) % P
    c = a * a % P
    a = 2 * a % P
    e = (c + 1) % P
    T = a * e % P
    X = a * b % P
    a = (1 - c) % P
    Y = e * a % P
    Z = a * b % P
    return X, Y, Z, T


# ---- the untwisted restatement (what the device computes) ---------------------------------------------------------------
def decode(b: bytes):
    """RFC 9496 decaf448 decode on the untwisted curve: affine (x, y) or None"""
    assert len(b) == 56
    s = int.from_bytes(b, "little")
    if s >= P or s & 1:
        return None
    ss = s * s % P
    u1 = (1 + ss) % P
    u2 = (u1 * u1 + 4 * NEG_D * ss) % P
    I, ok = isr(u2 * u1 * u1)
    if not ok:
        return None
    u3 = absv(2 * s * I * u1 * SQRT_MINUS_D)
    x = u3 * I * u2 * INV_SQRT_MINUS_D % P
    y = (1 - ss) * I * u1 % P
    return x, y


def encode_ext(X, Z, T) -> bytes:
    """RFC 9496 decaf448 encode of an untwisted extended point (X : Y : Z : T) (Y is not read)"""
    u1 = (X + T) * (X - T) % P
    I, _ = isr((1 - D) * u1 * X * X)
    r = absv(I * u1 * SQRT_MINUS_D)
    u2 = (r * Z * INV_SQRT_MINUS_D - T) % P
    s = absv((1 - D) * I * X * u2)
    return s.to_bytes(56, "little")


def encode(pt) -> bytes:
    x, y = pt
    return encode_ext(x, 1, x * y % P)


G0 = decode(GENERATOR_BYTES)


# ---- scalars --------------------------------------------------------------------------------------------------------------
def scalar_ok(k56: bytes) -> bool:
    """DecafScalar::from_canonical_bytes (decaf/scalar.rs:22-32)"""
    assert len(k56) == 56
    return (k56[55] >> 6) == 0 and int.from_bytes(k56, "little") < L


def enc_scalar(k: int) -> bytes:
    return k.to_bytes(56, "little")


def gen_scalar(k: int) -> int:
    """the Ed448 base-point scalar of [k]G: (-2 k) mod ell"""
    return (-2 * k) % L


# ---- the group entries ----------------------------------------------------------------------------------------------------
def mul(k56: bytes, p56: bytes) -> bytes:
    pt = decode(p56)
    assert pt is not None and scalar_ok(k56)
    return encode(M.mul(int.from_bytes(k56, "little"), pt))


def mul_gen(k56: bytes) -> bytes:
    assert scalar_ok(k56)
    return encode(M.mul(gen_scalar(int.from_bytes(k56, "little")), M.B))


def lincomb(ks, pts56) -> bytes:
    acc = M.IDENTITY
    for k56, p56 in zip(ks, pts56):
        acc = M.add(acc, M.mul(int.from_bytes(k56, "little"), decode(p56)))
    return encode(acc)


# ---- hashing --------------------------------------------------------------------------------------------------------------
def shake256(data: bytes, n: int) -> bytes:
    return hashlib.shake_256(data).digest(n)


def dst_prime(dst: bytes) -> bytes:
    """the DST as expand_message_xof absorbs it: over 255 bytes it is SHAKE256("H2C-OVERSIZE-DST-" || DST, 56)"""
    if not dst:
        raise ValueError("EmptyDst")
    return shake256(b"H2C-OVERSIZE-DST-" + dst, 56) if len(dst) > 255 else dst


def xof_suffix(dst: bytes, len_in_bytes: int) -> bytes:
    """what follows the message: I2OSP(len_in_bytes, 2) || DST' || I2OSP(len(DST'), 1)"""
    d = dst_prime(dst)
    return len_in_bytes.to_bytes(2, "big") + d + bytes([len(d)])


def expand_message_xof(msg: bytes, dst: bytes, len_in_bytes: int) -> bytes:
    return shake256(msg + xof_suffix(dst, len_in_bytes), len_in_bytes)


def hash_to_curve(msg: bytes, dst: bytes, nonuniform: bool = False) -> bytes:
    """hash_from_bytes (RO) / encode_from_bytes (NU) for Decaf448: field elements are 56 little-endian bytes mod p"""
    if nonuniform:
        u = expand_message_xof(msg, dst, 56)
        return tw_compress(tw_map(int.from_bytes(u, "little")))
    return from_uniform_bytes(expand_message_xof(msg, dst, 112))


def from_uniform_bytes(u: bytes) -> bytes:
    """DecafPoint::from_uniform_bytes then compress (decaf/points.rs:79-92): each 56-byte half little-endian mod p through
    the map, the two points added on the twisted curve"""
    assert len(u) == 112
    q0 = tw_map(int.from_bytes(u[:56], "little"))
    q1 = tw_map(int.from_bytes(u[56:], "little"))
    return tw_compress(tw_add(q0, q1))


def hash_to_scalar(msg: bytes, dst: bytes) -> bytes:
    """hash_to_scalar::<Decaf448, ExpandMsgXof<Shake256>, U64>: 64 little-endian bytes mod ell, to_repr"""
    u = expand_message_xof(msg, dst, 64)
    return (int.from_bytes(u, "little") % L).to_bytes(56, "little")
