// ecgpu.hpp — C++ host-side mirror of the reference's operator surface for the scalar-multiplication path,
// header-only, over the C ABI in include/ecgpu.h.  (The reference is Rust; this image has no Rust toolchain, so the
// host layer above the ABI is C++; INTEGRATION.md shows the equivalent Rust shim.)
//
// Names follow the reference's traits so that call sites read the same:
//   Engine::mul(points, scalars)                      <->  ProjectivePoint * Scalar            (k256/src/arithmetic/mul.rs:249-274)
//   Engine::mul_vartime(...)                          <->  MulVartime::mul_vartime             (mul.rs:276-295)   [same kernel]
//   Engine::mul_by_generator(scalars)                 <->  ProjectivePoint::mul_by_generator   (mul.rs:180-232)
//   Engine::lincomb(points, scalars)                  <->  LinearCombination::lincomb          (mul.rs:66-109)
//   Engine::mul_by_generator_and_mul_add_vartime(...) <->  MulByGeneratorVartime::...          (mul.rs:303-310)
//   Engine::batch_normalize(jacobian)                 <->  BatchNormalize::batch_normalize     (projective.rs:345-365)
//   Engine::hash_to_curve / encode_to_curve / hash_to_scalar <-> GroupDigest::hash_from_bytes / encode_from_bytes,
//                                                         hash2curve::hash_to_scalar (hash2curve/src/group_digest.rs:88-143)
//   Engine::x448(k, u)                                <->  x448::x448_unchecked / EphemeralSecret::diffie_hellman (x448/src/lib.rs)
//   Engine::ed448_verify(pk, sig, msgs, ctx, ph)      <->  ed448 VerifyingKey::verify_raw / verify_ctx / verify_prehashed
//   Engine::ed448_mul / ed448_mul_gen / ed448_lincomb <->  EdwardsPoint * EdwardsScalar, Group::mul_by_generator,
//                                                         LinearCombination::lincomb (ed448-goldilocks/src/edwards/extended.rs)
//   Engine::ed448_hash_to_curve / ed448_hash_to_scalar <-> GroupDigest for Ed448 (hash_from_bytes / encode_from_bytes),
//                                                         hash_to_scalar::<Ed448, ExpandMsgXof<Shake256>, U84>
//   Engine::decaf448_mul / decaf448_mul_gen / decaf448_lincomb / decaf448_check / decaf448_hash_to_curve /
//   decaf448_hash_to_scalar                          <->  DecafPoint * DecafScalar, GENERATOR * k, LinearCombination,
//                                                         CompressedDecaf::decompress, GroupDigest / hash_to_scalar for Decaf448
// The typed surface below is for the 256-bit curves with big-endian records (secp256k1, P-256, sm2, brainpoolP256r1/t1);
// the other curves of include/ecgpu.h (48 / 28 / 24-byte records, bign's little-endian records) are reached through the
// C ABI directly or the Python mirror, which sizes its buffers per curve.
// Fallible decoding mirrors CtOption/Result: out-of-range scalars / off-curve points throw DecodeError carrying the
// index of the first offender; arithmetic itself is total.
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/ecgpu.h"

namespace ecgpu {

using Scalar = std::array<uint8_t, 32>;  // big-endian, < n          (Scalar::to_bytes)
struct AffinePoint {                     // AffinePoint { x, y, infinity } (k256/src/arithmetic/affine.rs:37-49)
  std::array<uint8_t, 32> x{}, y{};
  uint8_t infinity = 0;
  static AffinePoint identity() {
    AffinePoint p;
    p.infinity = 1;
    return p;
  }
};
struct JacobianPoint {  // X, Y, Z big-endian; x = X/Z^2, y = Y/Z^3; Z = 0 is the identity
  std::array<uint8_t, 32> X{}, Y{}, Z{};
};
struct ProjectivePoint {  // the reference's own form: homogeneous, x = X/Z, y = Y/Z, identity (0:1:0)
  std::array<uint8_t, 32> X{}, Y{}, Z{};  // (k256/src/arithmetic/projective.rs:49-53)
};

struct Error : std::runtime_error {
  ecg_status code;
  Error(ecg_status c, const std::string& m) : std::runtime_error(m), code(c) {}
};
struct DecodeError : Error {  // Scalar::from_repr / AffinePoint::from_coordinates returned None in the reference
  size_t index;
  DecodeError(ecg_status c, const std::string& m, size_t i) : Error(c, m), index(i) {}
};

class Engine {
 public:
  // zeroize: clear the device-side copies of scalars, window tables and intermediates after every call
  // (ECG_FLAG_ZEROIZE; the reference zeroizes secrets on drop)
  // consttime: ECG_FLAG_CONSTTIME — scalar-independent table selects and sign folding, k*G through the variable-base
  // routine, per-term lincomb (the analogue of the reference's constant-time Mul; costs measured in bench.py configs.8)
  explicit Engine(ecg_curve curve, const std::vector<int>& devices = {0}, bool zeroize = false, bool consttime = false) : curve_(curve) {
    ecg_status st = ecg_ctx_create(devices.data(), (int)devices.size(), (zeroize ? ECG_FLAG_ZEROIZE : 0u) | (consttime ? ECG_FLAG_CONSTTIME : 0u), &ctx_);
    if (st != ECG_OK) throw Error(st, "ecg_ctx_create failed (no CUDA device? there is no CPU fallback)");
  }
  ~Engine() { ecg_ctx_destroy(ctx_); }
  Engine(const Engine&) = delete;
  Engine& operator=(const Engine&) = delete;

  std::vector<AffinePoint> mul(const std::vector<AffinePoint>& points, const std::vector<Scalar>& scalars) {
    size_t n = check_sizes(points.size(), scalars.size());
    pack(points);
    std::vector<uint8_t> out(64 * n), oinf(n);
    check(ecg_mul_batch(ctx_, curve_, n, flat(scalars), xy_.data(), inf_.data(), out.data(), oinf.data()));
    return unpack(out, oinf);
  }
  std::vector<AffinePoint> mul_vartime(const std::vector<AffinePoint>& p, const std::vector<Scalar>& k) { return mul(p, k); }

  std::vector<AffinePoint> mul_by_generator(const std::vector<Scalar>& scalars) {
    size_t n = scalars.size();
    std::vector<uint8_t> out(64 * n), oinf(n);
    check(ecg_mul_gen_batch(ctx_, curve_, n, flat(scalars), out.data(), oinf.data()));
    return unpack(out, oinf);
  }
  std::vector<AffinePoint> mul_by_generator_vartime(const std::vector<Scalar>& k) { return mul_by_generator(k); }

  AffinePoint lincomb(const std::vector<AffinePoint>& points, const std::vector<Scalar>& scalars) {
    size_t n = check_sizes(points.size(), scalars.size());
    pack(points);
    std::vector<uint8_t> out(64), oinf(1);
    check(ecg_lincomb(ctx_, curve_, n, flat(scalars), xy_.data(), inf_.data(), out.data(), oinf.data()));
    return unpack(out, oinf)[0];
  }
  AffinePoint lincomb_vartime(const std::vector<AffinePoint>& p, const std::vector<Scalar>& k) { return lincomb(p, k); }

  // a[i]*G + b[i]*P[i]
  std::vector<AffinePoint> mul_by_generator_and_mul_add_vartime(const std::vector<Scalar>& a, const std::vector<Scalar>& b,
                                                                const std::vector<AffinePoint>& points) {
    size_t n = check_sizes(points.size(), a.size());
    check_sizes(n, b.size());
    pack(points);
    std::vector<uint8_t> out(64 * n), oinf(n);
    check(ecg_mul_gen_add_batch(ctx_, curve_, n, flat(a), flat(b), xy_.data(), inf_.data(), out.data(), oinf.data()));
    return unpack(out, oinf);
  }

  std::vector<AffinePoint> batch_normalize(const std::vector<JacobianPoint>& pts) {
    size_t n = pts.size();
    std::vector<uint8_t> out(64 * n), oinf(n);
    check(ecg_batch_normalize(ctx_, curve_, n, reinterpret_cast<const uint8_t*>(pts.data()), out.data(), oinf.data()));
    return unpack(out, oinf);
  }

  // BatchNormalize::batch_normalize on the reference's homogeneous coordinates (projective.rs:367-391)
  std::vector<AffinePoint> batch_normalize(const std::vector<ProjectivePoint>& pts) {
    size_t n = pts.size();
    std::vector<uint8_t> out(64 * n), oinf(n);
    check(ecg_batch_normalize_hom(ctx_, curve_, n, reinterpret_cast<const uint8_t*>(pts.data()), out.data(), oinf.data()));
    return unpack(out, oinf);
  }
  // FieldElement::sqrt over a batch; ok[i] = false (and a zero root) where the input is not a square
  std::vector<std::array<uint8_t, 32>> field_sqrt(const std::vector<std::array<uint8_t, 32>>& a, std::vector<bool>* ok = nullptr) {
    size_t n = a.size();
    std::vector<std::array<uint8_t, 32>> r(n);
    std::vector<uint8_t> sq(n);
    check(ecg_field_sqrt_batch(ctx_, curve_, n, reinterpret_cast<const uint8_t*>(a.data()), reinterpret_cast<uint8_t*>(r.data()), sq.data()));
    if (ok) ok->assign(sq.begin(), sq.end());
    return r;
  }

  // ---- X448 (RFC 7748), 56-byte little-endian records; the same on an Engine of any curve ----
  using X448Bytes = std::array<uint8_t, 56>;
  // x448::x448_unchecked / EphemeralSecret::diffie_hellman over a batch (x448/src/lib.rs:25-31, :159-163); u empty: u = 5
  // for every scalar, the public keys (PublicKey::from).  ok (optional): ok[i] = false where u[i] is byte-for-byte one of
  // the low-order encodings x448::x448 refuses.  An all-zero result is returned, not refused (RFC 7748 section 6.2 leaves
  // that check to the protocol).
  std::vector<X448Bytes> x448(const std::vector<X448Bytes>& k, const std::vector<X448Bytes>& u = {}, std::vector<bool>* ok = nullptr) {
    size_t n = k.size();
    if (!u.empty()) check_sizes(n, u.size());
    std::vector<X448Bytes> r(n);
    std::vector<uint8_t> flags(n);
    check(ecg_x448_batch(ctx_, n, reinterpret_cast<const uint8_t*>(k.data()), u.empty() ? nullptr : reinterpret_cast<const uint8_t*>(u.data()),
                         reinterpret_cast<uint8_t*>(r.data()), flags.data()));
    if (ok) ok->assign(flags.begin(), flags.end());
    return r;
  }

  // ---- Ed448 (RFC 8032) verification, 57-byte keys and 114-byte signatures; the same on an Engine of any curve ----
  using Ed448Key = std::array<uint8_t, 57>;
  using Ed448Sig = std::array<uint8_t, 114>;
  // VerifyingKey::from_bytes(pk[i]) then verify_ctx(sig[i], context, msgs[i]) (verify_raw: empty context), or with
  // prehashed = true verify_prehashed with msgs[i] = PH(M) = SHAKE256(M, 64) (ed448-goldilocks/src/sign/verifying_key.rs:
  // 187-312); result[i] = true iff the reference accepts.  One context of at most 255 bytes for the whole call.
  std::vector<bool> ed448_verify(const std::vector<Ed448Key>& pk, const std::vector<Ed448Sig>& sig, const std::vector<std::vector<uint8_t>>& msgs,
                                 const std::vector<uint8_t>& context = {}, bool prehashed = false) {
    size_t n = pk.size();
    check_sizes(n, sig.size());
    check_sizes(n, msgs.size());
    std::vector<uint64_t> offsets(n + 1, 0);
    std::vector<uint8_t> data;
    for (size_t i = 0; i < n; i++) {
      data.insert(data.end(), msgs[i].begin(), msgs[i].end());
      offsets[i + 1] = data.size();
    }
    std::vector<uint8_t> valid(n);
    check(ecg_ed448_verify_batch(ctx_, n, reinterpret_cast<const uint8_t*>(pk.data()), reinterpret_cast<const uint8_t*>(sig.data()),
                                 data.empty() ? nullptr : data.data(), offsets.data(), context.empty() ? nullptr : context.data(),
                                 context.size(), prehashed ? 1 : 0, valid.data()));
    return std::vector<bool>(valid.begin(), valid.end());
  }

  // ---- Ed448 group operations, 57-byte scalars and compressed points; the same on an Engine of any curve ----
  using Ed448Scalar = std::array<uint8_t, 57>;
  using Ed448Point = std::array<uint8_t, 57>;
  // out[i] = [k[i]] P[i]: EdwardsPoint * EdwardsScalar (ed448-goldilocks/src/edwards/extended.rs:698-741)
  std::vector<Ed448Point> ed448_mul(const std::vector<Ed448Scalar>& k, const std::vector<Ed448Point>& P) {
    check_sizes(k.size(), P.size());
    std::vector<Ed448Point> out(k.size());
    check(ecg_ed448_mul_batch(ctx_, k.size(), reinterpret_cast<const uint8_t*>(k.data()), reinterpret_cast<const uint8_t*>(P.data()),
                              reinterpret_cast<uint8_t*>(out.data())));
    return out;
  }
  // out[i] = [k[i]] B: Group::mul_by_generator
  std::vector<Ed448Point> ed448_mul_gen(const std::vector<Ed448Scalar>& k) {
    std::vector<Ed448Point> out(k.size());
    check(ecg_ed448_mul_gen_batch(ctx_, k.size(), reinterpret_cast<const uint8_t*>(k.data()), reinterpret_cast<uint8_t*>(out.data())));
    return out;
  }
  // sum [k[i]] P[i]: LinearCombination::lincomb (empty input: the identity 01 00 .. 00)
  Ed448Point ed448_lincomb(const std::vector<Ed448Scalar>& k, const std::vector<Ed448Point>& P) {
    check_sizes(k.size(), P.size());
    Ed448Point out{};
    check(ecg_ed448_lincomb(ctx_, k.size(), reinterpret_cast<const uint8_t*>(k.data()), reinterpret_cast<const uint8_t*>(P.data()), out.data()));
    return out;
  }
  // hash_from_bytes (nonuniform = false) / encode_from_bytes for edwards448_XOF:SHAKE256_ELL2_{RO,NU}_ under one DST:
  // compressed points, valid inputs of ed448_mul
  std::vector<Ed448Point> ed448_hash_to_curve(const std::vector<std::vector<uint8_t>>& msgs, const std::vector<uint8_t>& dst,
                                              bool nonuniform = false) {
    std::vector<uint64_t> offsets;
    std::vector<uint8_t> data = pack(msgs, offsets);
    std::vector<Ed448Point> out(msgs.size());
    check(ecg_ed448_hash_to_curve_batch(ctx_, msgs.size(), data.empty() ? nullptr : data.data(), offsets.data(), dst.data(), dst.size(),
                                        nonuniform ? 1 : 0, reinterpret_cast<uint8_t*>(out.data())));
    return out;
  }
  // hash_to_scalar::<Ed448, ExpandMsgXof<Shake256>, U84>: 57-byte scalar records (byte 56 = 0)
  std::vector<Ed448Scalar> ed448_hash_to_scalar(const std::vector<std::vector<uint8_t>>& msgs, const std::vector<uint8_t>& dst) {
    std::vector<uint64_t> offsets;
    std::vector<uint8_t> data = pack(msgs, offsets);
    std::vector<Ed448Scalar> out(msgs.size());
    check(ecg_ed448_hash_to_scalar_batch(ctx_, msgs.size(), data.empty() ? nullptr : data.data(), offsets.data(), dst.data(), dst.size(),
                                         reinterpret_cast<uint8_t*>(out.data())));
    return out;
  }

  // ---- Decaf448 (RFC 9496), 56-byte scalars and encodings; the same on an Engine of any curve ----
  using Decaf448Bytes = std::array<uint8_t, 56>;
  // out[i] = [k[i]] P[i]: DecafPoint * DecafScalar
  std::vector<Decaf448Bytes> decaf448_mul(const std::vector<Decaf448Bytes>& k, const std::vector<Decaf448Bytes>& P) {
    check_sizes(k.size(), P.size());
    std::vector<Decaf448Bytes> out(k.size());
    check(ecg_decaf448_mul_batch(ctx_, k.size(), reinterpret_cast<const uint8_t*>(k.data()), reinterpret_cast<const uint8_t*>(P.data()),
                                 reinterpret_cast<uint8_t*>(out.data())));
    return out;
  }
  // out[i] = [k[i]] G (DecafPoint::GENERATOR)
  std::vector<Decaf448Bytes> decaf448_mul_gen(const std::vector<Decaf448Bytes>& k) {
    std::vector<Decaf448Bytes> out(k.size());
    check(ecg_decaf448_mul_gen_batch(ctx_, k.size(), reinterpret_cast<const uint8_t*>(k.data()), reinterpret_cast<uint8_t*>(out.data())));
    return out;
  }
  // sum [k[i]] P[i] (empty input: the identity, 56 zero bytes)
  Decaf448Bytes decaf448_lincomb(const std::vector<Decaf448Bytes>& k, const std::vector<Decaf448Bytes>& P) {
    check_sizes(k.size(), P.size());
    Decaf448Bytes out{};
    check(ecg_decaf448_lincomb(ctx_, k.size(), reinterpret_cast<const uint8_t*>(k.data()), reinterpret_cast<const uint8_t*>(P.data()), out.data()));
    return out;
  }
  // result[i] = true iff CompressedDecaf::decompress accepts P[i]
  std::vector<bool> decaf448_check(const std::vector<Decaf448Bytes>& P) {
    std::vector<uint8_t> ok(P.size());
    check(ecg_decaf448_check_batch(ctx_, P.size(), reinterpret_cast<const uint8_t*>(P.data()), ok.data()));
    return std::vector<bool>(ok.begin(), ok.end());
  }
  // hash_from_bytes (nonuniform = false) / encode_from_bytes for decaf448_XOF:SHAKE256_D448MAP_{RO,NU}_ under one DST
  std::vector<Decaf448Bytes> decaf448_hash_to_curve(const std::vector<std::vector<uint8_t>>& msgs, const std::vector<uint8_t>& dst,
                                                    bool nonuniform = false) {
    std::vector<uint64_t> offsets;
    std::vector<uint8_t> data = pack(msgs, offsets);
    std::vector<Decaf448Bytes> out(msgs.size());
    check(ecg_decaf448_hash_to_curve_batch(ctx_, msgs.size(), data.empty() ? nullptr : data.data(), offsets.data(), dst.data(), dst.size(),
                                           nonuniform ? 1 : 0, reinterpret_cast<uint8_t*>(out.data())));
    return out;
  }
  // hash_to_scalar::<Decaf448, ExpandMsgXof<Shake256>, U64>: 56-byte little-endian scalars
  std::vector<Decaf448Bytes> decaf448_hash_to_scalar(const std::vector<std::vector<uint8_t>>& msgs, const std::vector<uint8_t>& dst) {
    std::vector<uint64_t> offsets;
    std::vector<uint8_t> data = pack(msgs, offsets);
    std::vector<Decaf448Bytes> out(msgs.size());
    check(ecg_decaf448_hash_to_scalar_batch(ctx_, msgs.size(), data.empty() ? nullptr : data.data(), offsets.data(), dst.data(), dst.size(),
                                            reinterpret_cast<uint8_t*>(out.data())));
    return out;
  }

  // ---- widening (SURVEY 8(f)): verification, wire format, key agreement ----
  using Bytes32 = std::array<uint8_t, 32>;
  using Sig64 = std::array<uint8_t, 64>;
  using Sec1Compressed = std::array<uint8_t, 33>;

  // schnorr::VerifyingKey::verify_raw over a batch (k256/src/schnorr/verifying.rs:76-99); secp256k1 only
  std::vector<bool> schnorr_verify(const std::vector<Bytes32>& pk_x, const std::vector<Bytes32>& msg, const std::vector<Sig64>& sig) {
    size_t n = check_sizes(pk_x.size(), msg.size());
    check_sizes(n, sig.size());
    std::vector<uint8_t> valid(n);
    check(ecg_schnorr_verify_batch(ctx_, n, reinterpret_cast<const uint8_t*>(pk_x.data()), reinterpret_cast<const uint8_t*>(msg.data()),
                                   reinterpret_cast<const uint8_t*>(sig.data()), valid.data()));
    return std::vector<bool>(valid.begin(), valid.end());
  }
  // ecdsa::VerifyingKey::verify_prehash over a batch (k256/src/ecdsa.rs:93-121); low_s_only = EcdsaCurve::NORMALIZE_S
  std::vector<bool> ecdsa_verify_prehash(const std::vector<Bytes32>& z, const std::vector<Sig64>& sig, const std::vector<AffinePoint>& q,
                                         bool low_s_only) {
    size_t n = check_sizes(z.size(), sig.size());
    check_sizes(n, q.size());
    pack(q);
    std::vector<uint8_t> valid(n);
    check(ecg_ecdsa_verify_batch(ctx_, curve_, n, reinterpret_cast<const uint8_t*>(z.data()), reinterpret_cast<const uint8_t*>(sig.data()),
                                 xy_.data(), low_s_only ? 1 : 0, valid.data()));
    return std::vector<bool>(valid.begin(), valid.end());
  }
  // ecdsa::VerifyingKey::recover_from_prehash over a batch (k256/src/ecdsa.rs:45-88): recid = RecoveryId::to_byte per signature;
  // ok[i] = false (and an all-zero point) where recovery fails
  std::vector<AffinePoint> ecdsa_recover_prehash(const std::vector<Bytes32>& z, const std::vector<Sig64>& sig, const std::vector<uint8_t>& recid,
                                                 bool low_s_only, std::vector<bool>* ok = nullptr) {
    size_t n = check_sizes(z.size(), sig.size());
    check_sizes(n, recid.size());
    std::vector<uint8_t> out(64 * n), valid(n), noinf(n, 0);
    check(ecg_ecdsa_recover_batch(ctx_, curve_, n, reinterpret_cast<const uint8_t*>(z.data()), reinterpret_cast<const uint8_t*>(sig.data()),
                                  recid.data(), low_s_only ? 1 : 0, out.data(), valid.data()));
    if (ok) ok->assign(valid.begin(), valid.end());
    return unpack(out, noinf);
  }
  // sm2::dsa::VerifyingKey::verify_prehash over a batch (sm2/src/dsa/verifying.rs:138-175): e = SM3(Z_A || M) per signature
  std::vector<bool> sm2dsa_verify_prehash(const std::vector<Bytes32>& e, const std::vector<Sig64>& sig, const std::vector<AffinePoint>& q) {
    size_t n = check_sizes(e.size(), sig.size());
    check_sizes(n, q.size());
    pack(q);
    std::vector<uint8_t> valid(n);
    check(ecg_sm2dsa_verify_batch(ctx_, n, reinterpret_cast<const uint8_t*>(e.data()), reinterpret_cast<const uint8_t*>(sig.data()), xy_.data(),
                                  valid.data()));
    return std::vector<bool>(valid.begin(), valid.end());
  }
  // AffinePoint::decompress over a batch (primeorder/src/affine.rs:179-198); ok[i] = false where x is not on the curve
  std::vector<AffinePoint> decompress(const std::vector<Sec1Compressed>& rec, std::vector<bool>* ok = nullptr) {
    size_t n = rec.size();
    std::vector<uint8_t> out(64 * n), oinf(n), valid(n);
    check(ecg_decompress_batch(ctx_, curve_, n, reinterpret_cast<const uint8_t*>(rec.data()), out.data(), oinf.data(), valid.data()));
    if (ok) ok->assign(valid.begin(), valid.end());
    return unpack(out, oinf);
  }
  // to_sec1_point(true) / GroupEncoding::to_bytes (primeorder/src/affine.rs:387-402): byte layout only, no device work
  static Sec1Compressed compress(const AffinePoint& p) {
    Sec1Compressed r{};
    if (p.infinity) return r;  // identity = 33 zero bytes
    r[0] = 2 + (p.y[31] & 1);
    std::copy(p.x.begin(), p.x.end(), r.begin() + 1);
    return r;
  }
  // diffie_hellman (k256/src/ecdh.rs:46-60): x-coordinate of secret[i] * public[i], through ecg_mul_batch_x (y is never
  // formed).  VARIABLE TIME in the secret — the kernels index window tables by scalar digits and branch on exceptional
  // cases, the reference's diffie_hellman is constant time — hence the name; construct the Engine with zeroize = true.
  // Like the reference's NonZeroScalar / PublicKey inputs, a zero scalar, an identity peer or an identity result is an
  // error, never an all-zero shared secret.
  std::vector<Bytes32> diffie_hellman_vartime(const std::vector<Scalar>& secret, const std::vector<AffinePoint>& pub) {
    size_t n = check_sizes(pub.size(), secret.size());
    for (size_t i = 0; i < n; i++) {
      if (pub[i].infinity) throw DecodeError(ECG_EINVAL, "diffie_hellman_vartime: identity public key", i);
      if (std::all_of(secret[i].begin(), secret[i].end(), [](uint8_t b) { return b == 0; }))
        throw DecodeError(ECG_EINVAL, "diffie_hellman_vartime: zero secret scalar", i);
    }
    pack(pub);
    std::vector<Bytes32> r(n);
    std::vector<uint8_t> oinf(n);
    check(ecg_mul_batch_x(ctx_, curve_, n, flat(secret), xy_.data(), nullptr, reinterpret_cast<uint8_t*>(r.data()), oinf.data()));
    for (size_t i = 0; i < n; i++)
      if (oinf[i]) throw DecodeError(ECG_EINVAL, "diffie_hellman_vartime: identity shared point", i);
    return r;
  }
  // PublicKey::from_secret_scalar over a batch, SEC1-compressed.  VARIABLE TIME in the secret (see above).
  std::vector<Sec1Compressed> derive_public_keys_vartime(const std::vector<Scalar>& secret) {
    for (size_t i = 0; i < secret.size(); i++)
      if (std::all_of(secret[i].begin(), secret[i].end(), [](uint8_t b) { return b == 0; }))
        throw DecodeError(ECG_EINVAL, "derive_public_keys_vartime: zero secret scalar", i);
    std::vector<AffinePoint> p = mul_by_generator(secret);
    std::vector<Sec1Compressed> r(p.size());
    for (size_t i = 0; i < p.size(); i++) r[i] = compress(p[i]);
    return r;
  }

  // GroupDigest::hash_from_bytes (nonuniform = false) / encode_from_bytes (true) over a batch of messages, RFC 9380 with
  // expand_message_xmd<SHA-256> (hash2curve/src/group_digest.rs:88-118; suites of k256 / p256 arithmetic/hash2curve.rs)
  std::vector<AffinePoint> hash_to_curve(const std::vector<std::string>& msgs, const std::string& dst, bool nonuniform = false) {
    size_t n = msgs.size();
    std::vector<uint64_t> offs(n + 1, 0);
    std::string all;
    for (size_t i = 0; i < n; i++) {
      all += msgs[i];
      offs[i + 1] = all.size();
    }
    std::vector<uint8_t> out(64 * n), oinf(n);
    check(ecg_hash_to_curve_batch(ctx_, curve_, n, reinterpret_cast<const uint8_t*>(all.data()), offs.data(),
                                  reinterpret_cast<const uint8_t*>(dst.data()), dst.size(), nonuniform ? 1 : 0, out.data(), oinf.data()));
    return unpack(out, oinf);
  }
  std::vector<AffinePoint> encode_to_curve(const std::vector<std::string>& msgs, const std::string& dst) { return hash_to_curve(msgs, dst, true); }
  // hash2curve::hash_to_scalar over a batch (group_digest.rs:131-143, L = 48)
  std::vector<Scalar> hash_to_scalar(const std::vector<std::string>& msgs, const std::string& dst) {
    size_t n = msgs.size();
    std::vector<uint64_t> offs(n + 1, 0);
    std::string all;
    for (size_t i = 0; i < n; i++) {
      all += msgs[i];
      offs[i + 1] = all.size();
    }
    std::vector<Scalar> r(n);
    check(ecg_hash_to_scalar_batch(ctx_, curve_, n, reinterpret_cast<const uint8_t*>(all.data()), offs.data(),
                                   reinterpret_cast<const uint8_t*>(dst.data()), dst.size(), reinterpret_cast<uint8_t*>(r.data())));
    return r;
  }

  uint64_t kernel_launches() const { return ecg_kernel_launches(ctx_); }

 private:
  static size_t check_sizes(size_t a, size_t b) {
    if (a != b) throw Error(ECG_EINVAL, "points/scalars length mismatch");
    return a;
  }
  static const uint8_t* flat(const std::vector<Scalar>& s) { return reinterpret_cast<const uint8_t*>(s.data()); }
  // messages back to back and their n + 1 offsets (the layout of the message-taking entries)
  static std::vector<uint8_t> pack(const std::vector<std::vector<uint8_t>>& msgs, std::vector<uint64_t>& offsets) {
    std::vector<uint8_t> data;
    offsets.assign(msgs.size() + 1, 0);
    for (size_t i = 0; i < msgs.size(); i++) {
      data.insert(data.end(), msgs[i].begin(), msgs[i].end());
      offsets[i + 1] = data.size();
    }
    return data;
  }
  void pack(const std::vector<AffinePoint>& pts) {
    xy_.resize(64 * pts.size());
    inf_.resize(pts.size());
    for (size_t i = 0; i < pts.size(); i++) {
      std::copy(pts[i].x.begin(), pts[i].x.end(), xy_.begin() + 64 * i);
      std::copy(pts[i].y.begin(), pts[i].y.end(), xy_.begin() + 64 * i + 32);
      inf_[i] = pts[i].infinity;
    }
  }
  static std::vector<AffinePoint> unpack(const std::vector<uint8_t>& xy, const std::vector<uint8_t>& inf) {
    std::vector<AffinePoint> r(inf.size());
    for (size_t i = 0; i < r.size(); i++) {
      std::copy(xy.begin() + 64 * i, xy.begin() + 64 * i + 32, r[i].x.begin());
      std::copy(xy.begin() + 64 * i + 32, xy.begin() + 64 * i + 64, r[i].y.begin());
      r[i].infinity = inf[i];
    }
    return r;
  }
  void check(ecg_status st) {
    if (st == ECG_OK) return;
    std::string m = ecg_last_error(ctx_);
    if (st == ECG_ESCALAR_RANGE || st == ECG_ENOT_ON_CURVE) throw DecodeError(st, m, ecg_last_error_index(ctx_));
    throw Error(st, m);
  }
  ecg_curve curve_;
  ecg_ctx* ctx_ = nullptr;
  std::vector<uint8_t> xy_, inf_;
};

}  // namespace ecgpu
