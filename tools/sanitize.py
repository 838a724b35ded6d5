"""Small invocation of every C-ABI entry point, meant to be run under compute-sanitizer on the GPU box:
    compute-sanitizer --tool memcheck  --error-exitcode 9 python tools/sanitize.py
    compute-sanitizer --tool racecheck --error-exitcode 9 python tools/sanitize.py
    compute-sanitizer --tool initcheck --error-exitcode 9 python tools/sanitize.py
Sizes are tiny (the tools slow kernels 10-100x); results are still checked against the oracle port."""
import os, random, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "elliptic-curves_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
import ecgpu, pyref, ecref
from helpers import pack_scalars, pack_points, unpack_points

def main():
    eng = ecgpu.Engine()
    rng = random.Random(7)
    for curve in ("k256", "p256"):
        c = pyref.CURVES[curve]
        n = 300
        ks = [rng.randrange(c.n) for _ in range(n)]; ks[0] = 0; ks[1] = c.n - 1
        pts = [pyref.mul(c, rng.randrange(1, c.n), pyref.G(c)) for _ in range(n)]; pts[2] = None
        xy, inf = pack_points(pts)
        oxy, oinf = eng.mul_batch(curve, pack_scalars(ks), xy, inf)
        got = unpack_points(oxy, oinf)
        for i in range(0, n, 37):
            assert got[i] == pyref.mul(c, ks[i], pts[i]), (curve, "mul", i)
        gxy, ginf = eng.mul_by_generator(curve, pack_scalars(ks))
        got = unpack_points(gxy, ginf)
        for i in range(0, n, 37):
            assert got[i] == pyref.mul(c, ks[i], pyref.G(c)), (curve, "gen", i)
        for m in (5, 8200):   # per-term path and bucket-method path (>= 2^13 terms)
            kk = [rng.randrange(c.n) for _ in range(m)]
            pp = [pts[i % n] for i in range(m)]
            pxy, pinf = pack_points(pp)
            lxy, linf = eng.lincomb(curve, pack_scalars(kk), pxy, pinf)
            rxy, rinf = ecref.lincomb(curve, pack_scalars(kk), pxy, pinf, nthreads=8)
            assert np.array_equal(np.asarray(lxy).reshape(-1), np.asarray(rxy).reshape(-1)) and int(linf) == int(rinf), (curve, "lincomb", m)
        a = [rng.randrange(c.n) for _ in range(n)]
        mxy, minf = eng.mul_by_generator_and_mul_add(curve, pack_scalars(a), pack_scalars(ks), xy, inf)
        got = unpack_points(mxy, minf)
        for i in range(0, n, 41):
            assert got[i] == pyref.add(c, pyref.mul(c, a[i], pyref.G(c)), pyref.mul(c, ks[i], pts[i])), (curve, "mga", i)
        fa = pack_scalars([rng.randrange(c.p) for _ in range(n)]); fb = pack_scalars([rng.randrange(c.p) for _ in range(n)])
        for op in range(6):
            eng.field_op(curve, op, fa, fb)
        sec1 = np.zeros((n, 33), np.uint8)
        for i, P in enumerate(pts):
            if P is not None:
                sec1[i, 0] = 2 + (P[1] & 1); sec1[i, 1:] = np.frombuffer(P[0].to_bytes(32, "big"), np.uint8)
        eng.decompress_batch(curve, sec1)
        # ECDSA
        z = np.frombuffer(os.urandom(32 * 64), np.uint8).reshape(64, 32).copy()
        sig = np.zeros((64, 64), np.uint8); q = np.zeros((64, 64), np.uint8)
        for i in range(64):
            d = rng.randrange(1, c.n)
            r, s = pyref.ecdsa_sign(c, d, int.from_bytes(z[i].tobytes(), "big"), rng.randrange(1, c.n))
            sig[i] = np.frombuffer(r.to_bytes(32, "big") + s.to_bytes(32, "big"), np.uint8)
            Q = pyref.mul(c, d, pyref.G(c)); q[i] = np.frombuffer(Q[0].to_bytes(32, "big") + Q[1].to_bytes(32, "big"), np.uint8)
        v = eng.ecdsa_verify_batch(curve, z, sig, q, low_s_only=False)
        assert v.all(), (curve, "ecdsa")
    # BIP340
    c = pyref.CURVES["k256"]
    pk = np.zeros((64, 32), np.uint8); msg = np.frombuffer(os.urandom(32 * 64), np.uint8).reshape(64, 32).copy(); sg = np.zeros((64, 64), np.uint8)
    for i in range(64):
        d = rng.randrange(1, c.n)
        px, s64 = pyref.bip340_sign(d, msg[i].tobytes(), os.urandom(32))
        pk[i] = np.frombuffer(px, np.uint8); sg[i] = np.frombuffer(s64, np.uint8)
        assert pyref.bip340_verify(px, msg[i].tobytes(), s64)
    assert eng.schnorr_verify_batch(pk, msg, sg).all()
    # X448: a few pairs, low-order encodings among them, and the generator form
    import x448_model
    k448 = [os.urandom(56) for _ in range(16)]
    u448 = list(x448_model.LOW_ORDER) + [os.urandom(56) for _ in range(13)]
    out, ok = eng.x448(np.frombuffer(b"".join(k448), np.uint8), np.frombuffer(b"".join(u448), np.uint8))
    for i in range(16):
        assert out[i].tobytes() == x448_model.x448(k448[i], u448[i]) and ok[i] == x448_model.u_ok(u448[i]), ("x448", i)
    pub, _ = eng.x448(np.frombuffer(b"".join(k448[:4]), np.uint8))
    assert pub[0].tobytes() == x448_model.x448(k448[0], x448_model.GENERATOR)
    # Ed448: a few model-made signatures with a context, one empty message, one corrupted signature
    import ed448_model
    seed, ctx = os.urandom(57), b"sanitize"
    pk57 = ed448_model.public_key(seed)
    m448 = [b"", os.urandom(100), os.urandom(300)]
    s448 = [ed448_model.sign(seed, m, ctx) for m in m448]
    s448[2] = s448[2][:60] + bytes([s448[2][60] ^ 1]) + s448[2][61:]
    v = eng.ed448_verify(np.frombuffer(pk57 * 3, np.uint8), np.frombuffer(b"".join(s448), np.uint8), m448, ctx)
    assert list(v) == [1, 1, 0], ("ed448", list(v))
    # Ed448 group operations: one small call per entry, against the model
    import ed448_group_model
    kg = [rng.randrange(ed448_model.L) for _ in range(5)]
    K448 = np.frombuffer(b"".join(ed448_group_model.enc_scalar(k) for k in kg), np.uint8)
    P448 = np.frombuffer(pk57 * 5, np.uint8)
    g = eng.ed448_mul_gen(K448)
    assert [bytes(r) for r in g] == [ed448_group_model.mul_gen(ed448_group_model.enc_scalar(k)) for k in kg], "ed448 mul_gen"
    m = eng.ed448_mul(K448, P448)
    assert bytes(m[0]) == ed448_group_model.mul(ed448_group_model.enc_scalar(kg[0]), pk57), "ed448 mul"
    lc = eng.ed448_lincomb(K448, P448)
    assert bytes(lc) == ed448_group_model.lincomb([ed448_group_model.enc_scalar(k) for k in kg], [pk57] * 5), "ed448 lincomb"
    # Decaf448: one small call per entry, against the model
    import decaf448_model
    K56 = np.frombuffer(b"".join(decaf448_model.enc_scalar(k) for k in kg), np.uint8)
    dg = [bytes(r) for r in eng.decaf448_mul_gen(K56)]
    assert dg == [decaf448_model.mul_gen(decaf448_model.enc_scalar(k)) for k in kg], "decaf448 mul_gen"
    P56 = np.frombuffer(b"".join(dg), np.uint8)
    dm = eng.decaf448_mul(K56, P56)
    assert bytes(dm[0]) == decaf448_model.mul(decaf448_model.enc_scalar(kg[0]), dg[0]), "decaf448 mul"
    dl = eng.decaf448_lincomb(K56, P56)
    assert bytes(dl) == decaf448_model.lincomb([decaf448_model.enc_scalar(k) for k in kg], dg), "decaf448 lincomb"
    assert list(eng.decaf448_check(np.frombuffer(dg[0] + bytes([1]) * 56, np.uint8))) == [1, 0], "decaf448 check"
    dst = decaf448_model.HASH_TO_CURVE_ID
    assert [bytes(r) for r in eng.decaf448_hash_to_curve(m448, dst)] == [decaf448_model.hash_to_curve(m, dst) for m in m448], "decaf448 h2c"
    assert [bytes(r) for r in eng.decaf448_hash_to_curve(m448, bytes(300), True)] == [decaf448_model.hash_to_curve(m, bytes(300), True)
                                                                                      for m in m448], "decaf448 h2c nu"
    assert [bytes(r) for r in eng.decaf448_hash_to_scalar(m448, dst)] == [decaf448_model.hash_to_scalar(m, dst) for m in m448], "decaf448 h2s"
    eng.close()
    print("sanitize workload OK")

if __name__ == "__main__":
    main()
