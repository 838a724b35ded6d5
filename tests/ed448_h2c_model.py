"""Ed448 hash to curve (RFC 9380 edwards448_XOF:SHAKE256_ELL2_RO_ / _NU_) and hash to scalar in Python integers: the
model the Ed448 hashing tests check the device, its host twin and the C ABI against.  Two restatements live side by side.

The reference's own (ed448-goldilocks), literally:
  - ref_map: FieldElement::map_to_curve_elligator2 (field/element.rs:441-462): Z = -1, A = 156326, inv0, the
    unchecked square root y2^((p + 1) / 4) and the sign fix y = CMOV(-y, y, e2 xor sgn0(y));
  - ref_isogeny: AffinePoint::isogeny (edwards/affine.rs:75-104), each denominator inverted as inv0;
  - ref_add: EdwardsPoint::add (edwards/extended.rs:370-395), the unified extended addition; double is add(self);
  - to_affine (Z inverted as inv0) and AffinePoint::compress.
At u in {0, 1, p - 1} the map gives the Montgomery point (0, 0), the isogeny turns it into (0, 0) on edwards448 (not a
curve point), and the unified formulas keep X = Y = T = 0 through the additions: the output is 57 zero bytes.

The device's (ecg_ed448_h2c.cuh): the map straight-line with x = xn / xd kept as a fraction and one exponentiation,
the isogeny homogenised in xd into an extended point without inversion ((0 : 0 : 0 : 0) at the exceptional u), the
complete a = 1 formulas of ecg_ed448.cuh (add-2008-hwcd, dbl-2008-hwcd), Z set to 1 where it is 0, then the affine
compress of the normalisation kernel.

Field elements are read from 84 expanded bytes big-endian (Reduce<Array<u8, U84>>, field/element.rs:76-91); the
scalar likewise mod ell (edwards/scalar.rs:75-89), written as the 57-byte little-endian EdwardsScalar record."""
import hashlib

import ed448_model as M

P, L, D = M.P, M.L, M.D
A = 156326  # the Montgomery coefficient J of curve448
Z = P - 1
HASH_TO_CURVE_ID = b"edwards448_XOF:SHAKE256_ELL2_RO_"
ENCODE_TO_CURVE_ID = b"edwards448_XOF:SHAKE256_ELL2_NU_"
ZERO_RECORD = bytes(57)


def inv0(a):
    return pow(a % P, P - 2, P)


def sgn0(a):
    return (a % P) & 1


def reduce84(b: bytes) -> int:
    """Reduce<Array<u8, U84>> for FieldElement: big-endian mod p"""
    assert len(b) == 84
    return int.from_bytes(b, "big") % P


def reduce84_scalar(b: bytes) -> bytes:
    """Reduce<Array<u8, U84>> for EdwardsScalar, as the 57-byte record (to_bytes_rfc_8032; byte 56 = 0)"""
    assert len(b) == 84
    return (int.from_bytes(b, "big") % L).to_bytes(57, "little")


# ---- the reference's formulas -----------------------------------------------------------------------------------------
def ref_map(u):
    """map_to_curve_elligator2: the Montgomery point (x, y) of u"""
    t1 = Z * u * u % P
    e1 = t1 == P - 1
    if e1:
        t1 = 0
    x1 = inv0(t1 + 1)
    x1 = x1 * (P - A) % P
    gx1 = (x1 + A) * x1 % P
    gx1 = (gx1 + 1) * x1 % P
    x2 = (-x1 - A) % P
    gx2 = t1 * gx1 % P
    e2 = M.is_square(gx1)
    x = x1 if e2 else x2
    y2 = gx1 if e2 else gx2
    y = pow(y2, (P + 1) // 4, P)  # unchecked_sqrt
    if e2 ^ bool(sgn0(y)):
        y = (-y) % P
    return x, y


def ref_isogeny(pt):
    """AffinePoint::isogeny: the 4-isogeny from curve448 to edwards448, denominators inverted as inv0"""
    x, y = pt
    t0 = x * x % P
    t1 = (t0 + 1) % P
    t0 = (t0 - 1) % P
    t2 = 2 * y * y % P
    t3 = 2 * x % P
    x_num = 4 * t0 * y % P
    t5 = t0 * t0 % P
    x_den = (t5 + 2 * t2) % P
    t5 = t5 * x % P
    y_num = (t2 * t3 - t5) % P
    y_den = (t5 - t1 * t2) % P
    return x_num * inv0(x_den) % P, y_num * inv0(y_den) % P


def to_edwards(pt):
    x, y = pt
    return x, y, 1, x * y % P


def ref_add(p1, p2):
    """EdwardsPoint::add (a = 1): unified extended addition"""
    X1, Y1, Z1, T1 = p1
    X2, Y2, Z2, T2 = p2
    aXX = X1 * X2 % P
    dTT = D * T1 * T2 % P
    ZZ = Z1 * Z2 % P
    YY = Y1 * Y2 % P
    x1 = (X1 * Y2 + Y1 * X2) % P
    return (x1 * (ZZ - dTT) % P, (YY - aXX) * (ZZ + dTT) % P, (ZZ - dTT) * (ZZ + dTT) % P, (YY - aXX) * x1 % P)


def clear_cofactor(pt):
    pt = ref_add(pt, pt)
    return ref_add(pt, pt)


def compress_ext(pt) -> bytes:
    """to_affine (Z inverted as inv0) then AffinePoint::compress"""
    X, Y, Zc, _ = pt
    zi = inv0(Zc)
    return M.encode((X * zi % P, Y * zi % P))


def ref_point(u0, u1=None):
    """map(u0) (+ map(u1)), cleared of the cofactor, as the reference computes it"""
    q = to_edwards(ref_isogeny(ref_map(u0)))
    if u1 is not None:
        q = ref_add(q, to_edwards(ref_isogeny(ref_map(u1))))
    return clear_cofactor(q)


def ref_from_uniform(u: bytes) -> bytes:
    """84 bytes (one map, NU) or 168 bytes (two maps, RO) -> the compressed point"""
    if len(u) == 84:
        return compress_ext(ref_point(reduce84(u)))
    assert len(u) == 168
    return compress_ext(ref_point(reduce84(u[:84]), reduce84(u[84:])))


# ---- the device's formulas --------------------------------------------------------------------------------------------
def dev_map_parts(u):
    """the straight-line map: (X, D, y, e2, sgn0 of the root found) with the Montgomery x = X / D"""
    u %= P
    t1 = (-u * u) % P
    e1 = t1 == P - 1
    t1 = 0 if e1 else t1  # masked in the kernel
    xd = (1 + t1) % P
    xn = P - A  # x1 = -A / xd
    gxd = pow(xd, 3, P)
    gxn = (pow(xn, 3, P) + A * xn * xn * xd + xn * xd * xd) % P
    y1 = gxn * gxd * pow(gxn * pow(gxd, 3, P), (P - 3) // 4, P) % P
    e2 = y1 * y1 * gxd % P == gxn
    X = xn if e2 else xn * t1 % P  # x2 = -x1 - A = x1 t1
    y = y1 if e2 else y1 * u % P
    if e1:
        y = 0  # the y2 mask: the reference's t1 = 0 gives gx2 = 0
    s = sgn0(y)
    if e2 ^ bool(s):
        y = (-y) % P
    return X, xd, y, e2, s


def dev_map(u):
    """the map and the homogenised isogeny: the extended edwards448 point (xN yD : yN xD : xD yD : xN yN)"""
    X, Dd, y, _, _ = dev_map_parts(u)
    d2 = Dd * Dd % P
    y2 = y * y % P
    a = (X * X - d2) % P
    b = (X * X + d2) % P
    a2 = a * a % P
    yd4 = 4 * y2 * d2 * d2 % P
    xN = 4 * y * a * d2 % P
    xD = (a2 + yd4) % P
    yN = X * (yd4 - a2) % P
    yD = (a2 * X - 2 * y2 * b * d2 * Dd) % P
    return xN * yD % P, yN * xD % P, xD * yD % P, xN * yN % P


def dev_add(p, q):
    """ed_add of ecg_ed448.cuh (add-2008-hwcd, a = 1)"""
    X1, Y1, Z1, T1 = p
    X2, Y2, Z2, T2 = q
    a, b, c, dd = X1 * X2 % P, Y1 * Y2 % P, T1 * D * T2 % P, Z1 * Z2 % P
    e = ((X1 + Y1) * (X2 + Y2) - a - b) % P
    h, f, g = (b - a) % P, (dd - c) % P, (dd + c) % P
    return e * f % P, g * h % P, f * g % P, e * h % P


def dev_dbl(p):
    """ed_dbl of ecg_ed448.cuh (dbl-2008-hwcd, a = 1)"""
    X, Y, Zc, _ = p
    a, b, c = X * X % P, Y * Y % P, 2 * Zc * Zc % P
    e = ((X + Y) ** 2 - a - b) % P
    g, h = (a + b) % P, (a - b) % P
    f = (g - c) % P
    return e * f % P, g * h % P, f * g % P, e * h % P


def dev_point(u0, u1=None):
    q = dev_map(u0)
    if u1 is not None:
        q = dev_add(q, dev_map(u1))
    q = dev_dbl(dev_dbl(q))
    if q[2] == 0:  # the Z mask: (0 : 0 : 0 : 0) leaves as (0, 0), 57 zero bytes
        q = (q[0], q[1], 1, q[3])
    return q


def dev_from_uniform(u: bytes) -> bytes:
    if len(u) == 84:
        return compress_ext(dev_point(reduce84(u)))
    assert len(u) == 168
    return compress_ext(dev_point(reduce84(u[:84]), reduce84(u[84:])))


# ---- hashing ----------------------------------------------------------------------------------------------------------
def shake256(data: bytes, n: int) -> bytes:
    return hashlib.shake_256(data).digest(n)


def dst_prime(dst: bytes) -> bytes:
    """the DST as expand_message_xof absorbs it: over 255 bytes it is SHAKE256("H2C-OVERSIZE-DST-" || DST, 56)"""
    if not dst:
        raise ValueError("EmptyDst")
    return shake256(b"H2C-OVERSIZE-DST-" + dst, 56) if len(dst) > 255 else dst


def xof_suffix(dst: bytes, len_in_bytes: int) -> bytes:
    d = dst_prime(dst)
    return len_in_bytes.to_bytes(2, "big") + d + bytes([len(d)])


def expand_message_xof(msg: bytes, dst: bytes, len_in_bytes: int) -> bytes:
    return shake256(msg + xof_suffix(dst, len_in_bytes), len_in_bytes)


def hash_to_curve(msg: bytes, dst: bytes, nonuniform: bool = False, device_form: bool = False) -> bytes:
    """hash_from_bytes (RO) / encode_from_bytes (NU) for Ed448, compressed"""
    u = expand_message_xof(msg, dst, 84 if nonuniform else 168)
    return dev_from_uniform(u) if device_form else ref_from_uniform(u)


def hash_to_field(msg: bytes, dst: bytes):
    """the RO suite's u0, u1"""
    u = expand_message_xof(msg, dst, 168)
    return reduce84(u[:84]), reduce84(u[84:])


def hash_to_scalar(msg: bytes, dst: bytes) -> bytes:
    """hash_to_scalar::<Ed448, ExpandMsgXof<Shake256>, U84>"""
    return reduce84_scalar(expand_message_xof(msg, dst, 84))
