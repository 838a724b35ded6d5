"""ecgpu — Python (ctypes) host-side mirror of the reference's operator surface over libecgpu.so.

The shared library is the product; this module is the thinnest possible binding used by tests/ and
bench.py.  It mirrors the reference's names for the hot path:

    Engine.mul_batch(curve, k, P)              ProjectivePoint * Scalar over a batch     (k256/src/arithmetic/mul.rs:236-295)
    Engine.mul_by_generator(curve, k)          ProjectivePoint::mul_by_generator         (mul.rs:180-232)
    Engine.lincomb(curve, k, P)                LinearCombination::lincomb                (mul.rs:66-175)
    Engine.mul_by_generator_and_mul_add(...)   MulByGeneratorVartime::..._and_mul_add    (mul.rs:303-310)
    Engine.batch_normalize(curve, XYZ)         BatchNormalize::batch_normalize           (projective.rs:345-391)
    Engine.field_op(curve, op, a, b)           FieldElement add/sub/neg/mul/square/invert
    Engine.x448(k56, u56)                      x448::x448_unchecked / EphemeralSecret::diffie_hellman (x448/src/lib.rs)
    Engine.ed448_verify(pk57, sig114, msgs)    ed448 VerifyingKey::verify_raw / verify_ctx / verify_prehashed
    Engine.ed448_mul(k57, P57)                 EdwardsPoint * EdwardsScalar over a batch (edwards/extended.rs:698-741)
    Engine.ed448_mul_gen(k57)                  EdwardsPoint::mul_by_generator over a batch
    Engine.ed448_lincomb(k57, P57)             LinearCombination::lincomb for EdwardsPoint (extended.rs:310-312)
    Engine.decaf448_mul / _mul_gen / _lincomb  DecafPoint * DecafScalar, DecafPoint::GENERATOR * k, LinearCombination
    Engine.decaf448_check(P56)                 CompressedDecaf::decompress verdicts (decaf/points.rs:555-593)
    Engine.decaf448_hash_to_curve(msgs, dst)   hash_from_bytes / encode_from_bytes for Decaf448 (ExpandMsgXof<Shake256>)
    Engine.decaf448_hash_to_scalar(msgs, dst)  hash_to_scalar::<Decaf448, ExpandMsgXof<Shake256>, U64>

Buffers are numpy uint8 arrays (host mode) or raw device pointers (device mode, ECG_FLAG_DEVICE_PTRS).
There is NO CPU fallback: if libecgpu.so is missing, or no CUDA device is present, construction raises.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "libecgpu.so")

SECP256K1 = 0
NISTP256 = 1
NISTP384 = 2
SM2, BP256R1, BP256T1, BIGNP256, BP384R1, BP384T1, NISTP224, NISTP192, NISTP521 = 3, 4, 5, 6, 7, 8, 9, 10, 11
CURVE_IDS = {"k256": SECP256K1, "secp256k1": SECP256K1, "p256": NISTP256, "nistp256": NISTP256, "p384": NISTP384, "nistp384": NISTP384,
             "sm2": SM2, "bp256r1": BP256R1, "brainpoolp256r1": BP256R1, "bp256t1": BP256T1, "brainpoolp256t1": BP256T1,
             "bignp256": BIGNP256, "bp384r1": BP384R1, "brainpoolp384r1": BP384R1, "bp384t1": BP384T1, "brainpoolp384t1": BP384T1,
             "p224": NISTP224, "nistp224": NISTP224, "p192": NISTP192, "nistp192": NISTP192, "p521": NISTP521, "nistp521": NISTP521}
CURVE_IDS.update({i: i for i in range(12)})
# bytes per scalar / coordinate at the ABI (include/ecgpu.h)
FBYTES = {SECP256K1: 32, NISTP256: 32, NISTP384: 48, SM2: 32, BP256R1: 32, BP256T1: 32, BIGNP256: 32, BP384R1: 48, BP384T1: 48,
          NISTP224: 28, NISTP192: 24, NISTP521: 66}
# bign-curve256v1 records are little-endian (the reference's byte order for that curve); every other curve is big-endian
LITTLE_ENDIAN = {BIGNP256}

ECG_OK, ECG_EINVAL, ECG_ESCALAR_RANGE, ECG_ENOT_ON_CURVE, ECG_ECUDA, ECG_ENCCL, ECG_ENOMEM = range(7)
FLAG_DEVICE_PTRS = 1
FLAG_ZEROIZE = 2
FLAG_CONSTTIME = 4  # scalar-independent table selects / sign folding, k*G through the variable-base routine, per-term lincomb
FOP = {"add": 0, "sub": 1, "neg": 2, "mul": 3, "sqr": 4, "inv": 5}

EXPORTS = [
    "ecg_ctx_create", "ecg_ctx_destroy", "ecg_last_error", "ecg_last_error_index", "ecg_ctx_set_stream",
    "ecg_mul_batch", "ecg_mul_gen_batch", "ecg_lincomb", "ecg_lincomb_partial", "ecg_point_sum",
    "ecg_mul_gen_add_batch", "ecg_batch_normalize", "ecg_field_op_batch", "ecg_microbench",
    "ecg_kernel_launches", "ecg_version", "ecg_timing_enable", "ecg_timing_read",
    "ecg_schnorr_verify_batch", "ecg_ecdsa_verify_batch", "ecg_decompress_batch",
    "ecg_batch_normalize_hom", "ecg_mul_batch_x", "ecg_field_sqrt_batch",
    "ecg_hash_to_curve_batch", "ecg_hash_to_scalar_batch", "ecg_sm2dsa_verify_batch", "ecg_ecdsa_recover_batch",
    "ecg_x448_batch", "ecg_ed448_verify_batch", "ecg_ed448_mul_batch", "ecg_ed448_mul_gen_batch", "ecg_ed448_lincomb",
    "ecg_decaf448_mul_batch", "ecg_decaf448_mul_gen_batch", "ecg_decaf448_lincomb", "ecg_decaf448_check_batch",
    "ecg_decaf448_hash_to_curve_batch", "ecg_decaf448_hash_to_scalar_batch",
    "ecg_ed448_hash_to_curve_batch", "ecg_ed448_hash_to_scalar_batch",
]


class EcgError(RuntimeError):
    def __init__(self, code: int, msg: str, index: int = -1):
        super().__init__(f"ecgpu error {code}: {msg}" + (f" (first offending index {index})" if index >= 0 else ""))
        self.code = code
        self.index = index


class ScalarRangeError(EcgError):
    """Scalar::from_repr returned None in the reference (k >= n)."""


class NotOnCurveError(EcgError):
    """AffinePoint::from_coordinates returned None in the reference."""


_lib = None


def load_library(path: Optional[str] = None) -> ctypes.CDLL:
    """dlopen libecgpu.so (fails loudly if it has not been built: run `python -c 'import __graft_entry__ as g; g.build()'`)."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise FileNotFoundError(f"{p} not found: the CUDA extension is not built (no CPU fallback exists)")
    lib = ctypes.CDLL(p)
    vp, sz, u8p = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p
    lib.ecg_ctx_create.argtypes = [ctypes.POINTER(ctypes.c_int), ctypes.c_int, ctypes.c_uint, ctypes.POINTER(vp)]
    lib.ecg_ctx_create.restype = ctypes.c_int
    lib.ecg_ctx_destroy.argtypes = [vp]
    lib.ecg_ctx_destroy.restype = None
    lib.ecg_last_error.argtypes = [vp]
    lib.ecg_last_error.restype = ctypes.c_char_p
    lib.ecg_last_error_index.argtypes = [vp]
    lib.ecg_last_error_index.restype = sz
    lib.ecg_ctx_set_stream.argtypes = [vp, vp]
    lib.ecg_ctx_set_stream.restype = ctypes.c_int
    lib.ecg_mul_batch.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p, u8p, u8p]
    lib.ecg_mul_batch.restype = ctypes.c_int
    lib.ecg_mul_gen_batch.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p]
    lib.ecg_mul_gen_batch.restype = ctypes.c_int
    lib.ecg_lincomb.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p, u8p, u8p]
    lib.ecg_lincomb.restype = ctypes.c_int
    lib.ecg_lincomb_partial.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p, u8p]
    lib.ecg_lincomb_partial.restype = ctypes.c_int
    lib.ecg_point_sum.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p]
    lib.ecg_point_sum.restype = ctypes.c_int
    lib.ecg_mul_gen_add_batch.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p, u8p, u8p, u8p]
    lib.ecg_mul_gen_add_batch.restype = ctypes.c_int
    lib.ecg_batch_normalize.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p]
    lib.ecg_batch_normalize.restype = ctypes.c_int
    lib.ecg_field_op_batch.argtypes = [vp, ctypes.c_int, ctypes.c_int, sz, u8p, u8p, u8p]
    lib.ecg_field_op_batch.restype = ctypes.c_int
    lib.ecg_microbench.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double)]
    lib.ecg_microbench.restype = ctypes.c_int
    lib.ecg_kernel_launches.argtypes = [vp]
    lib.ecg_kernel_launches.restype = ctypes.c_uint64
    lib.ecg_timing_enable.argtypes = [vp, ctypes.c_int]
    lib.ecg_timing_enable.restype = ctypes.c_int
    lib.ecg_timing_read.argtypes = [vp, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_uint64)]
    lib.ecg_timing_read.restype = ctypes.c_int
    lib.ecg_schnorr_verify_batch.argtypes = [vp, sz, u8p, u8p, u8p, u8p]
    lib.ecg_schnorr_verify_batch.restype = ctypes.c_int
    lib.ecg_ecdsa_verify_batch.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p, ctypes.c_int, u8p]
    lib.ecg_ecdsa_verify_batch.restype = ctypes.c_int
    lib.ecg_sm2dsa_verify_batch.argtypes = [vp, sz, u8p, u8p, u8p, u8p]
    lib.ecg_ecdsa_recover_batch.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p, ctypes.c_int, u8p, u8p]
    lib.ecg_ecdsa_recover_batch.restype = ctypes.c_int
    lib.ecg_sm2dsa_verify_batch.restype = ctypes.c_int
    lib.ecg_decompress_batch.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p, u8p]
    lib.ecg_decompress_batch.restype = ctypes.c_int
    lib.ecg_batch_normalize_hom.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p]
    lib.ecg_batch_normalize_hom.restype = ctypes.c_int
    lib.ecg_mul_batch_x.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p, u8p, u8p]
    lib.ecg_mul_batch_x.restype = ctypes.c_int
    lib.ecg_field_sqrt_batch.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p]
    lib.ecg_field_sqrt_batch.restype = ctypes.c_int
    lib.ecg_hash_to_curve_batch.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p, sz, ctypes.c_int, u8p, u8p]
    lib.ecg_hash_to_curve_batch.restype = ctypes.c_int
    lib.ecg_hash_to_scalar_batch.argtypes = [vp, ctypes.c_int, sz, u8p, u8p, u8p, sz, u8p]
    lib.ecg_hash_to_scalar_batch.restype = ctypes.c_int
    lib.ecg_x448_batch.argtypes = [vp, sz, u8p, u8p, u8p, u8p]
    lib.ecg_x448_batch.restype = ctypes.c_int
    lib.ecg_ed448_verify_batch.argtypes = [vp, sz, u8p, u8p, u8p, u8p, u8p, sz, ctypes.c_int, u8p]
    lib.ecg_ed448_verify_batch.restype = ctypes.c_int
    lib.ecg_ed448_mul_batch.argtypes = [vp, sz, u8p, u8p, u8p]
    lib.ecg_ed448_mul_batch.restype = ctypes.c_int
    lib.ecg_ed448_mul_gen_batch.argtypes = [vp, sz, u8p, u8p]
    lib.ecg_ed448_mul_gen_batch.restype = ctypes.c_int
    lib.ecg_ed448_lincomb.argtypes = [vp, sz, u8p, u8p, u8p]
    lib.ecg_ed448_lincomb.restype = ctypes.c_int
    lib.ecg_ed448_hash_to_curve_batch.argtypes = [vp, sz, u8p, u8p, u8p, sz, ctypes.c_int, u8p]
    lib.ecg_ed448_hash_to_curve_batch.restype = ctypes.c_int
    lib.ecg_ed448_hash_to_scalar_batch.argtypes = [vp, sz, u8p, u8p, u8p, sz, u8p]
    lib.ecg_ed448_hash_to_scalar_batch.restype = ctypes.c_int
    lib.ecg_decaf448_mul_batch.argtypes = [vp, sz, u8p, u8p, u8p]
    lib.ecg_decaf448_mul_gen_batch.argtypes = [vp, sz, u8p, u8p]
    lib.ecg_decaf448_lincomb.argtypes = [vp, sz, u8p, u8p, u8p]
    lib.ecg_decaf448_check_batch.argtypes = [vp, sz, u8p, u8p]
    lib.ecg_decaf448_hash_to_curve_batch.argtypes = [vp, sz, u8p, u8p, u8p, sz, ctypes.c_int, u8p]
    lib.ecg_decaf448_hash_to_scalar_batch.argtypes = [vp, sz, u8p, u8p, u8p, sz, u8p]
    for f in ("mul_batch", "mul_gen_batch", "lincomb", "check_batch", "hash_to_curve_batch", "hash_to_scalar_batch"):
        getattr(lib, "ecg_decaf448_" + f).restype = ctypes.c_int
    lib.ecg_version.argtypes = []
    lib.ecg_version.restype = ctypes.c_char_p
    if path is None:
        _lib = lib
    return lib


def _u8(a, nbytes: int, name: str) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.uint8).reshape(-1)
    if a.size != nbytes:
        raise ValueError(f"{name}: expected {nbytes} bytes, got {a.size}")
    return a


def _out(a, nbytes: int, name: str) -> np.ndarray:
    """a caller-supplied output array is written in place by the library: it must be exactly what the ABI expects"""
    if a is None:
        return np.empty(nbytes, np.uint8)
    if not (isinstance(a, np.ndarray) and a.dtype == np.uint8 and a.flags["C_CONTIGUOUS"] and a.flags["WRITEABLE"] and a.size == nbytes):
        raise ValueError(f"{name}: expected a writable C-contiguous uint8 array of {nbytes} bytes")
    return a


def _ptr(a) -> ctypes.c_void_p:
    if a is None:
        return ctypes.c_void_p(0)
    if isinstance(a, np.ndarray):
        return ctypes.c_void_p(a.ctypes.data)
    return ctypes.c_void_p(int(a))  # raw device pointer


class Engine:
    """One ecg_ctx.  `devices=[0]` host-pointer mode by default; `device_ptrs=True` takes raw CUDA pointers."""

    def __init__(self, devices: Optional[Sequence[int]] = None, device_ptrs: bool = False, zeroize: bool = False, consttime: bool = False):
        self.lib = load_library()
        devs = list(devices) if devices else [0]
        arr = (ctypes.c_int * len(devs))(*devs)
        self._ctx = ctypes.c_void_p(0)
        self.device_ptrs = device_ptrs
        flags = (FLAG_DEVICE_PTRS if device_ptrs else 0) | (FLAG_ZEROIZE if zeroize else 0) | (FLAG_CONSTTIME if consttime else 0)
        rc = self.lib.ecg_ctx_create(arr, len(devs), flags, ctypes.byref(self._ctx))
        if rc != ECG_OK:
            raise EcgError(rc, "ecg_ctx_create failed (is a CUDA device visible? there is no CPU fallback)")

    def close(self):
        if getattr(self, "_ctx", None) and self._ctx.value:
            self.lib.ecg_ctx_destroy(self._ctx)
            self._ctx = ctypes.c_void_p(0)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc == ECG_OK:
            return
        msg = (self.lib.ecg_last_error(self._ctx) or b"").decode()
        idx = int(self.lib.ecg_last_error_index(self._ctx))
        if idx == 2**64 - 1:
            idx = -1
        if rc == ECG_ESCALAR_RANGE:
            raise ScalarRangeError(rc, msg, idx)
        if rc == ECG_ENOT_ON_CURVE:
            raise NotOnCurveError(rc, msg, idx)
        raise EcgError(rc, msg, idx)

    def set_stream(self, cuda_stream: int):
        """Run this ctx's work on the caller's CUDA stream (e.g. `torch.cuda.current_stream().cuda_stream`).  PyTorch's
        default stream has the handle 0, which the C ABI reads as "back to the ctx-owned stream": it is passed as
        cudaStreamLegacy (1), the explicit name of the same stream, so that the library's kernels are ordered with the
        producer of their inputs (a collective, a copy) instead of racing on a separate non-blocking stream."""
        if cuda_stream == 0:
            cuda_stream = 1  # cudaStreamLegacy
        self._check(self.lib.ecg_ctx_set_stream(self._ctx, ctypes.c_void_p(cuda_stream)))

    def reset_stream(self):
        self._check(self.lib.ecg_ctx_set_stream(self._ctx, ctypes.c_void_p(0)))

    @property
    def kernel_launches(self) -> int:
        return int(self.lib.ecg_kernel_launches(self._ctx))

    # ---- host-pointer API (numpy) ----
    def mul_batch(self, curve, k, P_xy, P_inf=None, out_xy=None, out_inf=None):
        c = CURVE_IDS[curve]
        fb = FBYTES[c]
        n = np.asarray(k).size // fb
        k = _u8(k, fb * n, "k")
        P_xy = _u8(P_xy, 2 * fb * n, "P_xy")
        if P_inf is not None:
            P_inf = _u8(P_inf, n, "P_inf")
        out_xy = _out(out_xy, 2 * fb * n, "out_xy")
        out_inf = _out(out_inf, n, "out_inf")
        self._check(self.lib.ecg_mul_batch(self._ctx, c, n, _ptr(k), _ptr(P_xy), _ptr(P_inf), _ptr(out_xy), _ptr(out_inf)))
        return out_xy.reshape(n, 2 * fb), out_inf

    def mul_by_generator(self, curve, k, out_xy=None, out_inf=None):
        c = CURVE_IDS[curve]
        fb = FBYTES[c]
        n = np.asarray(k).size // fb
        k = _u8(k, fb * n, "k")
        out_xy = _out(out_xy, 2 * fb * n, "out_xy")
        out_inf = _out(out_inf, n, "out_inf")
        self._check(self.lib.ecg_mul_gen_batch(self._ctx, c, n, _ptr(k), _ptr(out_xy), _ptr(out_inf)))
        return out_xy.reshape(n, 2 * fb), out_inf

    def mul_batch_x(self, curve, k, P_xy, P_inf=None):
        """x coordinate of k[i] * P[i] only (ecg_mul_batch_x) -> (x n x 32, inf)"""
        c = CURVE_IDS[curve]
        fb = FBYTES[c]
        n = np.asarray(k).size // fb
        k = _u8(k, fb * n, "k")
        P_xy = _u8(P_xy, 2 * fb * n, "P_xy")
        if P_inf is not None:
            P_inf = _u8(P_inf, n, "P_inf")
        out_x = np.empty(fb * n, np.uint8)
        out_inf = np.empty(n, np.uint8)
        self._check(self.lib.ecg_mul_batch_x(self._ctx, c, n, _ptr(k), _ptr(P_xy), _ptr(P_inf), _ptr(out_x), _ptr(out_inf)))
        return out_x.reshape(n, fb), out_inf

    def diffie_hellman_vartime(self, curve, secret_k, public_xy):
        """ECDH batch: x-coordinate of k[i] * P[i] (k256/src/ecdh.rs:46-60 `diffie_hellman`: `(public * secret).to_affine().x`).

        VARIABLE TIME in the secret: the kernels index window tables by scalar digits and branch on exceptional cases
        (INTEGRATION.md "constant time"); the reference's `diffie_hellman` is constant time.  Hence the name: use it
        only where timing of the device is not observable by an adversary, with an Engine(zeroize=True) so the staged
        scalars and tables are cleared after the call.  As in the reference, the inputs are a NonZeroScalar and a
        PublicKey: a zero scalar or an identity result is refused (ValueError) instead of yielding an all-zero secret."""
        fb = FBYTES[CURVE_IDS[curve]]
        n = np.asarray(secret_k).size // fb
        kk = _u8(secret_k, fb * n, "secret_k").reshape(n, fb)
        if n and not kk.any(axis=1).all():
            raise ValueError("diffie_hellman_vartime: zero secret scalar (the reference takes a NonZeroScalar)")
        out_x, out_inf = self.mul_batch_x(curve, kk, public_xy, None)
        if out_inf.any():
            raise ValueError("diffie_hellman_vartime: identity shared point")
        return out_x

    def lincomb(self, curve, k, P_xy, P_inf=None):
        c = CURVE_IDS[curve]
        fb = FBYTES[c]
        n = np.asarray(k).size // fb
        k = _u8(k, fb * n, "k")
        P_xy = _u8(P_xy, 2 * fb * n, "P_xy")
        if P_inf is not None:
            P_inf = _u8(P_inf, n, "P_inf")
        out_xy = np.zeros(2 * fb, np.uint8)
        out_inf = np.zeros(1, np.uint8)
        self._check(self.lib.ecg_lincomb(self._ctx, c, n, _ptr(k), _ptr(P_xy), _ptr(P_inf), _ptr(out_xy), _ptr(out_inf)))
        return out_xy, int(out_inf[0])

    def lincomb_partial(self, curve, k, P_xy, P_inf=None):
        c = CURVE_IDS[curve]
        fb = FBYTES[c]
        n = np.asarray(k).size // fb
        k = _u8(k, fb * n, "k")
        P_xy = _u8(P_xy, 2 * fb * n, "P_xy")
        if P_inf is not None:
            P_inf = _u8(P_inf, n, "P_inf")
        out = np.zeros(3 * fb, np.uint8)
        self._check(self.lib.ecg_lincomb_partial(self._ctx, c, n, _ptr(k), _ptr(P_xy), _ptr(P_inf), _ptr(out)))
        return out

    def point_sum(self, curve, xyz):
        c = CURVE_IDS[curve]
        xyz = np.ascontiguousarray(xyz, dtype=np.uint8).reshape(-1)
        m = xyz.size // (3 * FBYTES[c])
        out_xy = np.zeros(2 * FBYTES[c], np.uint8)
        out_inf = np.zeros(1, np.uint8)
        self._check(self.lib.ecg_point_sum(self._ctx, c, m, _ptr(xyz), _ptr(out_xy), _ptr(out_inf)))
        return out_xy, int(out_inf[0])

    def mul_by_generator_and_mul_add(self, curve, a, b, P_xy, P_inf=None):
        c = CURVE_IDS[curve]
        fb = FBYTES[c]
        n = np.asarray(a).size // fb
        a = _u8(a, fb * n, "a")
        b = _u8(b, fb * n, "b")
        P_xy = _u8(P_xy, 2 * fb * n, "P_xy")
        if P_inf is not None:
            P_inf = _u8(P_inf, n, "P_inf")
        out_xy = np.empty(2 * fb * n, np.uint8)
        out_inf = np.empty(n, np.uint8)
        self._check(self.lib.ecg_mul_gen_add_batch(self._ctx, c, n, _ptr(a), _ptr(b), _ptr(P_xy), _ptr(P_inf), _ptr(out_xy), _ptr(out_inf)))
        return out_xy.reshape(n, 2 * fb), out_inf

    @staticmethod
    def _pack_messages(msgs):
        """list of bytes -> (concatenated uint8 array, n + 1 uint64 offsets)"""
        offs = np.zeros(len(msgs) + 1, np.uint64)
        if len(msgs):
            offs[1:] = np.cumsum([len(m) for m in msgs], dtype=np.uint64)
        data = np.frombuffer(b"".join(bytes(m) for m in msgs), np.uint8).copy() if offs[-1] else np.zeros(1, np.uint8)
        return data, offs

    def hash_to_curve(self, curve, msgs, dst: bytes, nonuniform: bool = False):
        """GroupDigest::hash_from_bytes / encode_from_bytes over a batch of messages (hash2curve/src/group_digest.rs:88-118)
        -> (xy n x 64, inf)"""
        data, offs = self._pack_messages(msgs)
        return self.hash_to_curve_packed(curve, data, offs, dst, nonuniform)

    def hash_to_curve_packed(self, curve, data, offsets, dst: bytes, nonuniform: bool = False, out_xy=None, out_inf=None):
        """the same over messages already laid out as the C ABI takes them: `data` = the messages back to back (uint8),
        `offsets` = n + 1 uint64 byte offsets (message i = data[offsets[i]:offsets[i + 1]])"""
        c = CURVE_IDS[curve]
        offs = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = offs.size - 1
        if n < 0 or (n >= 0 and offs.size and int(offs[-1]) > np.asarray(data).size):
            raise ValueError("offsets: n + 1 ascending byte offsets into data")
        data = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
        if data.size == 0:
            data = np.zeros(1, np.uint8)
        d = np.frombuffer(bytes(dst), np.uint8).copy() if len(dst) else np.zeros(1, np.uint8)
        fb = FBYTES[c]
        out_xy = _out(out_xy, 2 * fb * n, "out_xy")
        out_inf = _out(out_inf, n, "out_inf")
        self._check(self.lib.ecg_hash_to_curve_batch(self._ctx, c, n, _ptr(data), _ptr(offs), _ptr(d), len(dst), 1 if nonuniform else 0,
                                                     _ptr(out_xy), _ptr(out_inf)))
        return out_xy.reshape(n, 2 * fb), out_inf

    def encode_to_curve(self, curve, msgs, dst: bytes):
        return self.hash_to_curve(curve, msgs, dst, nonuniform=True)

    def hash_to_scalar(self, curve, msgs, dst: bytes):
        """hash2curve::hash_to_scalar over a batch (group_digest.rs:131-143) -> n x 32 big-endian scalars"""
        c = CURVE_IDS[curve]
        n = len(msgs)
        data, offs = self._pack_messages(msgs)
        d = np.frombuffer(bytes(dst), np.uint8).copy() if len(dst) else np.zeros(1, np.uint8)
        fb = FBYTES[c]
        out = np.empty(fb * n, np.uint8)
        self._check(self.lib.ecg_hash_to_scalar_batch(self._ctx, c, n, _ptr(data), _ptr(offs), _ptr(d), len(dst), _ptr(out)))
        return out.reshape(n, fb)

    def schnorr_verify_batch(self, pk_x, msg32, sig64):
        """BIP340: VerifyingKey::verify_raw over a batch (k256/src/schnorr/verifying.rs:76-99) -> uint8 flags"""
        n = np.asarray(pk_x).size // 32
        pk_x = _u8(pk_x, 32 * n, "pk_x")
        msg32 = _u8(msg32, 32 * n, "msg32")
        sig64 = _u8(sig64, 64 * n, "sig64")
        valid = np.zeros(n, np.uint8)
        self._check(self.lib.ecg_schnorr_verify_batch(self._ctx, n, _ptr(pk_x), _ptr(msg32), _ptr(sig64), _ptr(valid)))
        return valid

    def ecdsa_verify_batch(self, curve, z32, sig64, Q_xy, low_s_only=False):
        """ECDSA verify_prehash over a batch -> uint8 flags.  Records are FB bytes (the curve's FieldBytes): z = the prehash
        after bits2field, signature r || s, public key x || y."""
        c = CURVE_IDS[curve]
        fb = FBYTES[c]
        n = np.asarray(z32).size // fb
        z32 = _u8(z32, fb * n, "z")
        sig64 = _u8(sig64, 2 * fb * n, "sig")
        Q_xy = _u8(Q_xy, 2 * fb * n, "Q_xy")
        valid = np.zeros(n, np.uint8)
        self._check(self.lib.ecg_ecdsa_verify_batch(self._ctx, c, n, _ptr(z32), _ptr(sig64), _ptr(Q_xy), 1 if low_s_only else 0, _ptr(valid)))
        return valid

    def ecdsa_recover_batch(self, curve, z32, sig64, recid, low_s_only=False, out_xy=None, valid=None):
        """VerifyingKey::recover_from_prehash over a batch (secp256k1 / P-256) -> (Q_xy n x 64, valid): prehash, r || s, one
        RecoveryId byte (bit 0: y of R odd, bit 1: x of R = r + n) per signature"""
        c = CURVE_IDS[curve]
        n = np.asarray(recid).size
        z32 = _u8(z32, 32 * n, "z")
        sig64 = _u8(sig64, 64 * n, "sig")
        recid = _u8(recid, n, "recid")
        out_xy = _out(out_xy, 64 * n, "out_xy")
        valid = _out(valid, n, "valid")
        self._check(self.lib.ecg_ecdsa_recover_batch(self._ctx, c, n, _ptr(z32), _ptr(sig64), _ptr(recid), 1 if low_s_only else 0,
                                                     _ptr(out_xy), _ptr(valid)))
        return out_xy.reshape(n, 64), valid

    def sm2dsa_verify_batch(self, e32, sig64, Q_xy):
        """SM2DSA verify_prehash over a batch -> uint8 flags: e = SM3(Z_A || M) (32 bytes), signature r || s, public key x || y"""
        n = np.asarray(e32).size // 32
        e32 = _u8(e32, 32 * n, "e")
        sig64 = _u8(sig64, 64 * n, "sig")
        Q_xy = _u8(Q_xy, 64 * n, "Q_xy")
        valid = np.zeros(n, np.uint8)
        self._check(self.lib.ecg_sm2dsa_verify_batch(self._ctx, n, _ptr(e32), _ptr(sig64), _ptr(Q_xy), _ptr(valid)))
        return valid

    def decompress_batch(self, curve, sec1_33):
        """AffinePoint::decompress over a batch of (1 + FB)-byte SEC1 compressed records -> (xy, inf, valid)"""
        c = CURVE_IDS[curve]
        fb = FBYTES[c]
        n = np.asarray(sec1_33).size // (fb + 1)
        sec1_33 = _u8(sec1_33, (fb + 1) * n, "sec1")
        out_xy = np.empty(2 * fb * n, np.uint8)
        out_inf = np.empty(n, np.uint8)
        valid = np.empty(n, np.uint8)
        self._check(self.lib.ecg_decompress_batch(self._ctx, c, n, _ptr(sec1_33), _ptr(out_xy), _ptr(out_inf), _ptr(valid)))
        return out_xy.reshape(n, 2 * fb), out_inf, valid

    @staticmethod
    def sec1_compress(xy, inf=None):
        """`GroupEncoding::to_bytes` / `to_sec1_point(true)` for a batch of affine outputs (primeorder/src/affine.rs:387-402):
        33-byte records, tag 02/03 by the parity of y then x; the identity is 33 zero bytes.  Pure byte shuffling on
        the host — the arithmetic (normalisation) already happened on the device."""
        xy = np.ascontiguousarray(xy, dtype=np.uint8).reshape(-1, 64)
        out = np.zeros((xy.shape[0], 33), np.uint8)
        out[:, 0] = 2 + (xy[:, 63] & 1)
        out[:, 1:] = xy[:, :32]
        if inf is not None:
            out[np.asarray(inf).reshape(-1) != 0] = 0
        return out

    def derive_public_keys_vartime(self, curve, secret_k, compressed=True):
        """Public-key derivation batch: `PublicKey::from_secret_scalar` = k * G, SEC1-encoded (SURVEY 8(f) rank 3;
        k256/src/schnorr/signing.rs:151 does the same for BIP340 keys).  Returns (records, inf).  VARIABLE TIME in the
        secret (table gathers by scalar digit) — see diffie_hellman_vartime; zero scalars are refused like NonZeroScalar."""
        n = np.asarray(secret_k).size // 32
        kk = _u8(secret_k, 32 * n, "secret_k").reshape(n, 32)
        if n and not kk.any(axis=1).all():
            raise ValueError("derive_public_keys_vartime: zero secret scalar (the reference takes a NonZeroScalar)")
        xy, inf = self.mul_by_generator(curve, secret_k)
        if compressed:
            return self.sec1_compress(xy, inf), inf
        out = np.zeros((xy.shape[0], 65), np.uint8)
        out[:, 0] = 4
        out[:, 1:] = xy
        out[inf != 0] = 0
        return out, inf

    def batch_normalize(self, curve, xyz):
        c = CURVE_IDS[curve]
        xyz = np.ascontiguousarray(xyz, dtype=np.uint8).reshape(-1)
        fb = FBYTES[c]
        n = xyz.size // (3 * fb)
        out_xy = np.empty(2 * fb * n, np.uint8)
        out_inf = np.empty(n, np.uint8)
        self._check(self.lib.ecg_batch_normalize(self._ctx, c, n, _ptr(xyz), _ptr(out_xy), _ptr(out_inf)))
        return out_xy.reshape(n, 2 * fb), out_inf

    def batch_normalize_hom(self, curve, xyz):
        """BatchNormalize for the reference's own homogeneous (X:Y:Z), x = X/Z (ecg_batch_normalize_hom)"""
        c = CURVE_IDS[curve]
        xyz = np.ascontiguousarray(xyz, dtype=np.uint8).reshape(-1)
        fb = FBYTES[c]
        n = xyz.size // (3 * fb)
        out_xy = np.empty(2 * fb * n, np.uint8)
        out_inf = np.empty(n, np.uint8)
        self._check(self.lib.ecg_batch_normalize_hom(self._ctx, c, n, _ptr(xyz), _ptr(out_xy), _ptr(out_inf)))
        return out_xy.reshape(n, 2 * fb), out_inf

    def field_sqrt(self, curve, a):
        """FieldElement::sqrt over a batch -> (roots n x FB, is_square)"""
        c = CURVE_IDS[curve]
        fb = FBYTES[c]
        n = np.asarray(a).size // fb
        a = _u8(a, fb * n, "a")
        out = np.empty(fb * n, np.uint8)
        ok = np.empty(n, np.uint8)
        self._check(self.lib.ecg_field_sqrt_batch(self._ctx, c, n, _ptr(a), _ptr(out), _ptr(ok)))
        return out.reshape(n, fb), ok

    def field_op(self, curve, op, a, b=None):
        c = CURVE_IDS[curve]
        fb = FBYTES[c]
        n = np.asarray(a).size // fb
        a = _u8(a, fb * n, "a")
        if b is not None:
            b = _u8(b, fb * n, "b")
        out = np.empty(fb * n, np.uint8)
        self._check(self.lib.ecg_field_op_batch(self._ctx, c, FOP[op] if isinstance(op, str) else op, n, _ptr(a), _ptr(b), _ptr(out)))
        return out.reshape(n, fb)

    def x448(self, k56, u56=None, out=None, ok=None):
        """X448 (RFC 7748) over a batch -> (out n x 56, ok n): out[i] = X448(k[i], u[i]) (x448::x448_unchecked); u56=None:
        u = 5, the public keys of the secrets (PublicKey::from).  ok[i] = 0 iff u[i] is byte-for-byte one of the
        low-order encodings x448::x448 refuses.  An all-zero out[i] (RFC 7748 section 6.2) is not refused here: compare
        with zero bytes where the protocol asks for it."""
        n = np.asarray(k56).size // 56
        k56 = _u8(k56, 56 * n, "k56")
        if u56 is not None:
            u56 = _u8(u56, 56 * n, "u56")
        out = _out(out, 56 * n, "out")
        ok = _out(ok, n, "ok")
        self._check(self.lib.ecg_x448_batch(self._ctx, n, _ptr(k56), _ptr(u56), _ptr(out), _ptr(ok)))
        return out.reshape(n, 56), ok

    def ed448_verify(self, pk57, sig114, msgs, context: bytes = b"", prehashed: bool = False):
        """Ed448 (RFC 8032) verification over a batch -> valid (n uint8): VerifyingKey::from_bytes(pk57[i]) and then
        verify_ctx(sig114[i], context, msgs[i]) (verify_raw: context b""), or with prehashed=True verify_prehashed with
        msgs[i] = PH(M) = SHAKE256(M, 64) as the caller computed it.  One context (<= 255 bytes) for the whole call."""
        data, offs = self._pack_messages(msgs)
        return self.ed448_verify_packed(pk57, sig114, data, offs, context, prehashed)

    def ed448_verify_packed(self, pk57, sig114, data, offsets, context: bytes = b"", prehashed: bool = False, valid=None):
        """the same over messages already laid out as the C ABI takes them: `data` = the messages back to back (uint8),
        `offsets` = n + 1 uint64 byte offsets (message i = data[offsets[i]:offsets[i + 1]])"""
        offs = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = offs.size - 1
        if n < 0 or int(offs[-1]) > np.asarray(data).size:
            raise ValueError("offsets: n + 1 ascending byte offsets into data")
        data = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
        if data.size == 0:
            data = np.zeros(1, np.uint8)
        pk57 = _u8(pk57, 57 * n, "pk57")
        sig114 = _u8(sig114, 114 * n, "sig114")
        ctx = np.frombuffer(bytes(context), np.uint8).copy() if len(context) else None
        valid = _out(valid, n, "valid")
        self._check(self.lib.ecg_ed448_verify_batch(self._ctx, n, _ptr(pk57), _ptr(sig114), _ptr(data), _ptr(offs), _ptr(ctx), len(context),
                                                    1 if prehashed else 0, _ptr(valid)))
        return valid

    def ed448_mul(self, k57, P57, out=None):
        """Ed448 group: out[i] = [k[i]] P[i] (n x 57 compressed records; EdwardsPoint * EdwardsScalar).  Scalars are 57-byte
        little-endian, accepted iff bytes 0..55 < ell (ScalarRangeError with the smallest index otherwise); points are
        compressed Edwards y, accepted iff CompressedEdwardsY::decompress accepts them (NotOnCurveError otherwise)."""
        n = np.asarray(k57).size // 57
        k57 = _u8(k57, 57 * n, "k57")
        P57 = _u8(P57, 57 * n, "P57")
        out = _out(out, 57 * n, "out")
        self._check(self.lib.ecg_ed448_mul_batch(self._ctx, n, _ptr(k57), _ptr(P57), _ptr(out)))
        return out.reshape(n, 57)

    def ed448_mul_gen(self, k57, out=None):
        """Ed448 group: out[i] = [k[i]] B (EdwardsPoint::mul_by_generator), n x 57 compressed records"""
        n = np.asarray(k57).size // 57
        k57 = _u8(k57, 57 * n, "k57")
        out = _out(out, 57 * n, "out")
        self._check(self.lib.ecg_ed448_mul_gen_batch(self._ctx, n, _ptr(k57), _ptr(out)))
        return out.reshape(n, 57)

    def ed448_lincomb(self, k57, P57):
        """Ed448 group: sum_i [k[i]] P[i] as one 57-byte compressed record (n = 0: the identity 01 00 .. 00)"""
        n = np.asarray(k57).size // 57
        k57 = _u8(k57, 57 * n, "k57")
        P57 = _u8(P57, 57 * n, "P57")
        out = np.empty(57, np.uint8)
        self._check(self.lib.ecg_ed448_lincomb(self._ctx, n, _ptr(k57), _ptr(P57), _ptr(out)))
        return out

    def ed448_hash_to_curve(self, msgs, dst: bytes, nonuniform: bool = False):
        """Ed448 hash_from_bytes (RO) / encode_from_bytes (NU) with ExpandMsgXof<Shake256> -> n x 57 compressed records,
        valid P57 inputs of ed448_mul"""
        data, offs = self._pack_messages(msgs)
        return self.ed448_hash_to_curve_packed(data, offs, dst, nonuniform)

    def ed448_hash_to_curve_packed(self, data, offsets, dst: bytes, nonuniform: bool = False, out=None):
        """the same over messages already laid out as the C ABI takes them (data + n + 1 uint64 offsets)"""
        offs = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = offs.size - 1
        if n < 0 or int(offs[-1]) > np.asarray(data).size:
            raise ValueError("offsets: n + 1 ascending byte offsets into data")
        data = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
        if data.size == 0:
            data = np.zeros(1, np.uint8)
        d = np.frombuffer(bytes(dst), np.uint8).copy() if len(dst) else np.zeros(1, np.uint8)
        out = _out(out, 57 * n, "out")
        self._check(self.lib.ecg_ed448_hash_to_curve_batch(self._ctx, n, _ptr(data), _ptr(offs), _ptr(d), len(dst), 1 if nonuniform else 0,
                                                           _ptr(out)))
        return out.reshape(n, 57)

    def ed448_hash_to_scalar(self, msgs, dst: bytes):
        """hash_to_scalar::<Ed448, ExpandMsgXof<Shake256>, U84> over a batch -> n x 57 scalar records (byte 56 = 0), valid
        k57 inputs of the Ed448 group entries"""
        n = len(msgs)
        data, offs = self._pack_messages(msgs)
        d = np.frombuffer(bytes(dst), np.uint8).copy() if len(dst) else np.zeros(1, np.uint8)
        out = np.empty(57 * n, np.uint8)
        self._check(self.lib.ecg_ed448_hash_to_scalar_batch(self._ctx, n, _ptr(data), _ptr(offs), _ptr(d), len(dst), _ptr(out)))
        return out.reshape(n, 57)

    def decaf448_mul(self, k56, P56, out=None):
        """Decaf448: out[i] = [k[i]] P[i] (n x 56 encodings; DecafPoint * DecafScalar).  Scalars are 56-byte little-endian,
        accepted iff DecafScalar::from_canonical_bytes accepts them (ScalarRangeError with the smallest index otherwise);
        points are accepted iff CompressedDecaf::decompress accepts them (NotOnCurveError otherwise)."""
        n = np.asarray(k56).size // 56
        k56 = _u8(k56, 56 * n, "k56")
        P56 = _u8(P56, 56 * n, "P56")
        out = _out(out, 56 * n, "out")
        self._check(self.lib.ecg_decaf448_mul_batch(self._ctx, n, _ptr(k56), _ptr(P56), _ptr(out)))
        return out.reshape(n, 56)

    def decaf448_mul_gen(self, k56, out=None):
        """Decaf448: out[i] = [k[i]] G (DecafPoint::GENERATOR), n x 56 encodings"""
        n = np.asarray(k56).size // 56
        k56 = _u8(k56, 56 * n, "k56")
        out = _out(out, 56 * n, "out")
        self._check(self.lib.ecg_decaf448_mul_gen_batch(self._ctx, n, _ptr(k56), _ptr(out)))
        return out.reshape(n, 56)

    def decaf448_lincomb(self, k56, P56):
        """Decaf448: sum_i [k[i]] P[i] as one 56-byte encoding (n = 0: the identity, 56 zero bytes)"""
        n = np.asarray(k56).size // 56
        k56 = _u8(k56, 56 * n, "k56")
        P56 = _u8(P56, 56 * n, "P56")
        out = np.empty(56, np.uint8)
        self._check(self.lib.ecg_decaf448_lincomb(self._ctx, n, _ptr(k56), _ptr(P56), _ptr(out)))
        return out

    def decaf448_check(self, P56, ok=None):
        """Decaf448: ok[i] = 1 iff CompressedDecaf::decompress accepts P[i] (verdicts, never an error)"""
        n = np.asarray(P56).size // 56
        P56 = _u8(P56, 56 * n, "P56")
        ok = _out(ok, n, "ok")
        self._check(self.lib.ecg_decaf448_check_batch(self._ctx, n, _ptr(P56), _ptr(ok)))
        return ok

    def decaf448_hash_to_curve(self, msgs, dst: bytes, nonuniform: bool = False):
        """Decaf448 hash_from_bytes (RO) / encode_from_bytes (NU) with ExpandMsgXof<Shake256> -> n x 56 encodings"""
        data, offs = self._pack_messages(msgs)
        return self.decaf448_hash_to_curve_packed(data, offs, dst, nonuniform)

    def decaf448_hash_to_curve_packed(self, data, offsets, dst: bytes, nonuniform: bool = False, out=None):
        """the same over messages already laid out as the C ABI takes them (data + n + 1 uint64 offsets)"""
        offs = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = offs.size - 1
        if n < 0 or int(offs[-1]) > np.asarray(data).size:
            raise ValueError("offsets: n + 1 ascending byte offsets into data")
        data = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
        if data.size == 0:
            data = np.zeros(1, np.uint8)
        d = np.frombuffer(bytes(dst), np.uint8).copy() if len(dst) else np.zeros(1, np.uint8)
        out = _out(out, 56 * n, "out")
        self._check(self.lib.ecg_decaf448_hash_to_curve_batch(self._ctx, n, _ptr(data), _ptr(offs), _ptr(d), len(dst), 1 if nonuniform else 0,
                                                              _ptr(out)))
        return out.reshape(n, 56)

    def decaf448_hash_to_scalar(self, msgs, dst: bytes):
        """hash_to_scalar::<Decaf448, ExpandMsgXof<Shake256>, U64> over a batch -> n x 56 little-endian scalars"""
        n = len(msgs)
        data, offs = self._pack_messages(msgs)
        d = np.frombuffer(bytes(dst), np.uint8).copy() if len(dst) else np.zeros(1, np.uint8)
        out = np.empty(56 * n, np.uint8)
        self._check(self.lib.ecg_decaf448_hash_to_scalar_batch(self._ctx, n, _ptr(data), _ptr(offs), _ptr(d), len(dst), _ptr(out)))
        return out.reshape(n, 56)

    # ---- raw-pointer API (device_ptrs=True): all arguments are integer CUDA device addresses ----
    def mul_batch_ptr(self, curve, n, k, P_xy, P_inf, out_xy, out_inf):
        self._check(self.lib.ecg_mul_batch(self._ctx, CURVE_IDS[curve], n, _ptr(k), _ptr(P_xy), _ptr(P_inf), _ptr(out_xy), _ptr(out_inf)))

    def mul_gen_batch_ptr(self, curve, n, k, out_xy, out_inf):
        self._check(self.lib.ecg_mul_gen_batch(self._ctx, CURVE_IDS[curve], n, _ptr(k), _ptr(out_xy), _ptr(out_inf)))

    def lincomb_partial_ptr(self, curve, n, k, P_xy, P_inf, out_xyz):
        self._check(self.lib.ecg_lincomb_partial(self._ctx, CURVE_IDS[curve], n, _ptr(k), _ptr(P_xy), _ptr(P_inf), _ptr(out_xyz)))

    def lincomb_ptr(self, curve, n, k, P_xy, P_inf, out_xy, out_inf):
        self._check(self.lib.ecg_lincomb(self._ctx, CURVE_IDS[curve], n, _ptr(k), _ptr(P_xy), _ptr(P_inf), _ptr(out_xy), _ptr(out_inf)))

    def mul_batch_x_ptr(self, curve, n, k, P_xy, P_inf, out_x, out_inf):
        self._check(self.lib.ecg_mul_batch_x(self._ctx, CURVE_IDS[curve], n, _ptr(k), _ptr(P_xy), _ptr(P_inf), _ptr(out_x), _ptr(out_inf)))

    def batch_normalize_ptr(self, curve, n, xyz, out_xy, out_inf):
        self._check(self.lib.ecg_batch_normalize(self._ctx, CURVE_IDS[curve], n, _ptr(xyz), _ptr(out_xy), _ptr(out_inf)))

    def batch_normalize_hom_ptr(self, curve, n, xyz, out_xy, out_inf):
        self._check(self.lib.ecg_batch_normalize_hom(self._ctx, CURVE_IDS[curve], n, _ptr(xyz), _ptr(out_xy), _ptr(out_inf)))

    def point_sum_ptr(self, curve, m, xyz, out_xy, out_inf):
        """sum of m Jacobian points (m*96 bytes in device memory, e.g. an all_gather receive buffer) -> affine, on the device"""
        self._check(self.lib.ecg_point_sum(self._ctx, CURVE_IDS[curve], m, _ptr(xyz), _ptr(out_xy), _ptr(out_inf)))

    def schnorr_verify_ptr(self, n, pk_x, msg32, sig64, valid):
        self._check(self.lib.ecg_schnorr_verify_batch(self._ctx, n, _ptr(pk_x), _ptr(msg32), _ptr(sig64), _ptr(valid)))

    def x448_ptr(self, n, k56, u56, out56, ok):
        """ecg_x448_batch on device buffers (u56 = 0: the generator; ok = 0: no flags)"""
        self._check(self.lib.ecg_x448_batch(self._ctx, n, _ptr(k56), _ptr(u56), _ptr(out56), _ptr(ok)))

    def ed448_verify_ptr(self, n, pk57, sig114, msgs, offsets, valid, context: bytes = b"", prehashed: bool = False):
        """ecg_ed448_verify_batch on device buffers (offsets: n + 1 uint64, 8-byte aligned); the context is host bytes"""
        ctx = np.frombuffer(bytes(context), np.uint8).copy() if len(context) else None
        self._check(self.lib.ecg_ed448_verify_batch(self._ctx, n, _ptr(pk57), _ptr(sig114), _ptr(msgs), _ptr(offsets), _ptr(ctx), len(context),
                                                    1 if prehashed else 0, _ptr(valid)))

    def ed448_mul_ptr(self, n, k57, P57, out57):
        """ecg_ed448_mul_batch on device buffers (57-byte records at any alignment)"""
        self._check(self.lib.ecg_ed448_mul_batch(self._ctx, n, _ptr(k57), _ptr(P57), _ptr(out57)))

    def ed448_mul_gen_ptr(self, n, k57, out57):
        """ecg_ed448_mul_gen_batch on device buffers"""
        self._check(self.lib.ecg_ed448_mul_gen_batch(self._ctx, n, _ptr(k57), _ptr(out57)))

    def ed448_lincomb_ptr(self, n, k57, P57, out57):
        """ecg_ed448_lincomb on device buffers (out57: 57 bytes)"""
        self._check(self.lib.ecg_ed448_lincomb(self._ctx, n, _ptr(k57), _ptr(P57), _ptr(out57)))

    def ed448_hash_to_curve_ptr(self, n, msgs, offsets, out57, dst: bytes, nonuniform: bool = False):
        """ecg_ed448_hash_to_curve_batch on device buffers (offsets: n + 1 uint64, 8-byte aligned; records at any alignment);
        the DST is host bytes"""
        d = np.frombuffer(bytes(dst), np.uint8).copy() if len(dst) else np.zeros(1, np.uint8)
        self._check(self.lib.ecg_ed448_hash_to_curve_batch(self._ctx, n, _ptr(msgs), _ptr(offsets), _ptr(d), len(dst), 1 if nonuniform else 0,
                                                           _ptr(out57)))

    def ed448_hash_to_scalar_ptr(self, n, msgs, offsets, out57, dst: bytes):
        """ecg_ed448_hash_to_scalar_batch on device buffers; the DST is host bytes"""
        d = np.frombuffer(bytes(dst), np.uint8).copy() if len(dst) else np.zeros(1, np.uint8)
        self._check(self.lib.ecg_ed448_hash_to_scalar_batch(self._ctx, n, _ptr(msgs), _ptr(offsets), _ptr(d), len(dst), _ptr(out57)))

    def decaf448_mul_ptr(self, n, k56, P56, out56):
        """ecg_decaf448_mul_batch on device buffers (56-byte records, 4-byte aligned)"""
        self._check(self.lib.ecg_decaf448_mul_batch(self._ctx, n, _ptr(k56), _ptr(P56), _ptr(out56)))

    def decaf448_mul_gen_ptr(self, n, k56, out56):
        """ecg_decaf448_mul_gen_batch on device buffers"""
        self._check(self.lib.ecg_decaf448_mul_gen_batch(self._ctx, n, _ptr(k56), _ptr(out56)))

    def decaf448_lincomb_ptr(self, n, k56, P56, out56):
        """ecg_decaf448_lincomb on device buffers (out56: 56 bytes)"""
        self._check(self.lib.ecg_decaf448_lincomb(self._ctx, n, _ptr(k56), _ptr(P56), _ptr(out56)))

    def decaf448_check_ptr(self, n, P56, ok):
        """ecg_decaf448_check_batch on device buffers"""
        self._check(self.lib.ecg_decaf448_check_batch(self._ctx, n, _ptr(P56), _ptr(ok)))

    def decaf448_hash_to_curve_ptr(self, n, msgs, offsets, out56, dst: bytes, nonuniform: bool = False):
        """ecg_decaf448_hash_to_curve_batch on device buffers (offsets: n + 1 uint64, 8-byte aligned); the DST is host bytes"""
        d = np.frombuffer(bytes(dst), np.uint8).copy() if len(dst) else np.zeros(1, np.uint8)
        self._check(self.lib.ecg_decaf448_hash_to_curve_batch(self._ctx, n, _ptr(msgs), _ptr(offsets), _ptr(d), len(dst), 1 if nonuniform else 0,
                                                              _ptr(out56)))

    def decaf448_hash_to_scalar_ptr(self, n, msgs, offsets, out56, dst: bytes):
        """ecg_decaf448_hash_to_scalar_batch on device buffers; the DST is host bytes"""
        d = np.frombuffer(bytes(dst), np.uint8).copy() if len(dst) else np.zeros(1, np.uint8)
        self._check(self.lib.ecg_decaf448_hash_to_scalar_batch(self._ctx, n, _ptr(msgs), _ptr(offsets), _ptr(d), len(dst), _ptr(out56)))

    def timing_enable(self, on: bool = True):
        self._check(self.lib.ecg_timing_enable(self._ctx, 1 if on else 0))

    def timing_read(self):
        """(accumulated ms of the dominant kernel, number of calls) since timing_enable"""
        ms = ctypes.c_double(0)
        calls = ctypes.c_uint64(0)
        self._check(self.lib.ecg_timing_read(self._ctx, ctypes.byref(ms), ctypes.byref(calls)))
        return ms.value, int(calls.value)

    def microbench(self, which: int, iters: int = 2000):
        ops = ctypes.c_double(0)
        ms = ctypes.c_double(0)
        self._check(self.lib.ecg_microbench(self._ctx, which, iters, ctypes.byref(ops), ctypes.byref(ms)))
        return ops.value, ms.value
