"""The Ed448 group operations (EdwardsPoint of ed448-goldilocks) in Python integers: the model the group tests check the
device, its host twin and OpenSSL against.  The curve arithmetic is ed448_model's.

What the reference does, entry by entry:
  - scalars are 57-byte little-endian records accepted iff EdwardsScalar::from_repr = from_canonical_bytes accepts them
    (edwards/scalar.rs:32-42).  Its test is (byte 56 == 0 | byte 55 >> 6 == 0) & (bytes 0..55 < ell); since
    ell < 2^446, "bytes 0..55 < ell" already forces byte 55 >> 6 == 0, so byte 56 is ignored and the rule is
    "bytes 0..55, read as an integer, < ell" (scalar_ok);
  - points are 57-byte records accepted iff GroupEncoding::from_bytes = CompressedEdwardsY::decompress accepts them
    (edwards/affine.rs:487-520): y = bytes 0..55 mod p, the sign of x in bit 7 of byte 56, on the curve, torsion free.
    The identity is accepted under either sign bit; (0, -1) and the all-zero record (y = 0: (+-1, 0), order 4) are not
    (decompress);
  - outputs are AffinePoint::compress (edwards/affine.rs:29-41), ed448_model.encode; the identity is 01 00 .. 00;
  - the reference's scalar_mul computes [4 (s / 4 mod ell)]P through the 4-isogeny (edwards/extended.rs:357-365)
    (reference_scalar_mul).  On the prime-order subgroup that is [s]P, and only such points pass the decoder, so a
    kernel may use any correct algorithm (the tests check the equivalence on subgroup points)."""
import ed448_model as M

P, L, D = M.P, M.L, M.D
IDENTITY_BYTES = bytes([1]) + bytes(56)


def scalar_ok(k57: bytes) -> bool:
    assert len(k57) == 57
    return int.from_bytes(k57[:56], "little") < L


def from_canonical_bytes(k57: bytes) -> bool:
    """the reference's test as written (edwards/scalar.rs:32-42); scalar_ok is its simplification"""
    valid = k57[56] == 0 or (k57[55] >> 6) == 0
    return valid and int.from_bytes(k57[:56], "little") < L


def scalar(k57: bytes) -> int:
    return int.from_bytes(k57[:56], "little")


def decompress(b57: bytes):
    """CompressedEdwardsY::decompress: the point, or None; the identity is accepted"""
    return M.decompress(b57)


def reference_scalar_mul(s: int, pt):
    """[4 (s / 4 mod ell)] pt, the reference's scalar_mul through the isogeny"""
    return M.mul(4 * (s * pow(4, -1, L) % L), pt)


def mul(k57: bytes, p57: bytes) -> bytes:
    pt = decompress(p57)
    assert pt is not None and scalar_ok(k57)
    return M.encode(M.mul(scalar(k57) % L, pt))


def mul_gen(k57: bytes) -> bytes:
    assert scalar_ok(k57)
    return M.encode(M.mul(scalar(k57), M.B))


def lincomb(ks, pts57) -> bytes:
    acc = M.IDENTITY
    for k57, p57 in zip(ks, pts57):
        acc = M.add(acc, M.mul(scalar(k57), decompress(p57)))
    return M.encode(acc)


def secret_scalar(seed: bytes) -> int:
    """the clamped SHAKE256(seed) scalar of RFC 8032 key generation, reduced mod ell (public key = its multiple of B)"""
    return M.expand_secret(seed)[0] % L


def enc_scalar(k: int, byte56: int = 0) -> bytes:
    return k.to_bytes(56, "little") + bytes([byte56])


def fixed_base_table(w: int, nd: int):
    """the fixed-base table: window i, entry j = (2j + 1) 2^(w i) B as (x, y, d x y), 42 little-endian 32-bit words per
    entry, entries of window i at 2^(w - 1) i .. ; -> bytes"""
    out = []
    bi = M.B
    for _ in range(nd):
        b2 = M.add(bi, bi)
        e = bi
        for _ in range(1 << (w - 1)):
            x, y = e
            out.append(x.to_bytes(56, "little") + y.to_bytes(56, "little") + (D * x * y % P).to_bytes(56, "little"))
            e = M.add(e, b2)
        for _ in range(w):
            bi = M.add(bi, bi)
    return b"".join(out)
