"""X448 (RFC 7748) in Python integers: the model the X448 tests check the device and its host twin against.

It follows the reference (x448/src/lib.rs, ed448-goldilocks/src/montgomery.rs): decodeScalar448 clamps and does not
reduce mod the group order, u is reduced mod p, the ladder is Costello-Smith Algorithm 8 over all 448 bits, and the
result is U * W^(p-2) (the identity gives 0).  The low-order byte check that x448::x448 adds on top of x448_unchecked is
a separate function, as it is a separate output of ecg_x448_batch."""

P = 2**448 - 2**224 - 1
A24 = 39082  # (A + 2) / 4, A = 156326
GENERATOR = (5).to_bytes(56, "little")
# MontgomeryPoint::LOW_A / LOW_B / LOW_C: the encodings of 0, 1 and p - 1
LOW_ORDER = (bytes(56), (1).to_bytes(56, "little"), (P - 1).to_bytes(56, "little"))


def decode_scalar(k: bytes) -> int:
    b = bytearray(k)
    assert len(b) == 56
    b[0] &= 252
    b[55] |= 128
    return int.from_bytes(b, "little")


def decode_u(u: bytes) -> int:
    assert len(u) == 56
    return int.from_bytes(u, "little") % P


def encode_u(x: int) -> bytes:
    return (x % P).to_bytes(56, "little")


def ladder_step(x2, z2, x3, z3, u):
    """differential_add_and_double: ((x2 : z2), (x3 : z3)) -> (2 (x2 : z2), (x2 : z2) + (x3 : z3)) with difference u, mod p"""
    t0, t1, t2, t3 = (x2 + z2) % P, (x2 - z2) % P, (x3 + z3) % P, (x3 - z3) % P
    t4, t5 = t0 * t0 % P, t1 * t1 % P
    t6 = (t4 - t5) % P
    t7, t8 = t0 * t3 % P, t1 * t2 % P
    t11, t12 = (t7 + t8) ** 2 % P, (t7 - t8) ** 2 % P
    return t4 * t5 % P, t6 * (A24 * t6 + t5) % P, t11, u * t12 % P


def x448_int(k: int, u: int) -> int:
    """the ladder on a decoded scalar and u (any integers; u is reduced mod p)"""
    u %= P
    x2, z2, x3, z3, swap = 1, 0, u, 1, 0
    for t in reversed(range(448)):
        bit = (k >> t) & 1
        if swap ^ bit:
            x2, x3, z2, z3 = x3, x2, z3, z2
        swap = bit
        x2, z2, x3, z3 = ladder_step(x2, z2, x3, z3, u)
    if swap:
        x2, z2 = x3, z3
    return x2 * pow(z2, P - 2, P) % P


def x448(k: bytes, u: bytes) -> bytes:
    """x448::x448_unchecked / EphemeralSecret::diffie_hellman: 56 bytes out, 56 zero bytes at the identity"""
    return encode_u(x448_int(decode_scalar(k), decode_u(u)))


def u_ok(u: bytes) -> bool:
    """False exactly when x448::x448 refuses u: its bytes are one of LOW_A, LOW_B, LOW_C"""
    return bytes(u) not in LOW_ORDER
