"""The batch driver of the per-element entries (ecgpu.cu: run_chunked) with two shards on one GPU.

ecg_ctx_create takes a device id more than once, so Engine([0, 0]) splits every batch into two contiguous shards that
run on the same device, each cut into whole-wave chunks and interleaved chunk by chunk on the two lanes, as they would on
two GPUs.  For one entry of each family (secp256k1 variable base, X448, Ed448 verification, Ed448 k*B from the
fixed-base table), at sizes that give each shard three chunks: the output equals a one-shard ctx's byte for byte, a
refused record in the second shard is reported with its index in the whole batch, and each call counts once in the
kernel timing."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _sizes(per_sm):
    """(n, wave): each of two shards is 3 waves + 5 elements, which chunk_schedule cuts into w, w and w + 5"""
    import torch

    wave = torch.cuda.get_device_properties(0).multi_processor_count * per_sm
    return 2 * (3 * wave + 5), wave


def _k256(n):
    import pyref
    from helpers import pack_points, random_points

    rng = np.random.default_rng(256)
    k = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    k[:, 0] &= 0x7F  # < 2^255 < n
    xy, inf = pack_points(random_points(pyref.CURVES["k256"], 16, seed=256))
    xy = np.tile(np.asarray(xy).reshape(16, 64), (n // 16 + 1, 1))[:n].copy()
    inf = np.tile(inf, n // 16 + 1)[:n].copy()

    def run(e, k_):
        out_xy, out_inf = e.mul_batch("k256", k_, xy, inf)
        return np.concatenate([np.asarray(out_xy).reshape(-1), out_inf])

    def refuse(k_, i):
        k_[i] = 0xFF  # >= n
    return k, run, refuse


def _x448(n):
    rng = np.random.default_rng(448)
    k = rng.integers(0, 256, (n, 56), dtype=np.uint8)
    u = rng.integers(0, 256, (n, 56), dtype=np.uint8)

    def run(e, k_):
        out, ok = e.x448(k_, u)
        return np.concatenate([np.asarray(out).reshape(-1), ok])
    return k, run, None


def _ed448_verify(n):
    """16 OpenSSL signatures over messages of 0 to 300 bytes, every fourth with a flipped bit in S, repeated"""
    from cryptography.hazmat.primitives.asymmetric.ed448 import Ed448PrivateKey

    rng = random.Random(57)
    base, want = [], []
    for j in range(16):
        sk = Ed448PrivateKey.from_private_bytes(rng.getrandbits(456).to_bytes(57, "little"))
        msg = rng.getrandbits(8 * 20 * j).to_bytes(20 * j, "little") if j else b""
        sig = bytearray(sk.sign(msg))
        if j % 4 == 3:
            sig[57 + j] ^= 1
        base.append((sk.public_key().public_bytes_raw(), bytes(sig), msg))
        want.append(int(j % 4 != 3))
    idx = [i % 16 for i in range(n)]
    pk = np.frombuffer(b"".join(base[j][0] for j in idx), np.uint8).copy()
    sig = np.frombuffer(b"".join(base[j][1] for j in idx), np.uint8).copy()
    data = np.frombuffer(b"".join(base[j][2] for j in idx), np.uint8).copy()
    offs = np.concatenate([[0], np.cumsum([len(base[j][2]) for j in idx])]).astype(np.uint64)

    def run(e, pk_):
        valid = e.ed448_verify_packed(pk_, sig, data, offs)
        assert list(valid) == [want[j] for j in idx]
        return valid
    return pk, run, None


def _ed448_mul_gen(n):
    rng = np.random.default_rng(4480)
    k = rng.integers(0, 256, (n, 57), dtype=np.uint8)
    k[:, 55] &= 0x1F  # < 2^445 < ell
    k[:, 56] = 0

    def run(e, k_):
        return e.ed448_mul_gen(k_)

    def refuse(k_, i):
        k_[i, :56] = 0xFF  # >= ell
    return k, run, refuse


# entry -> (elements per SM in one wave of its kernel, inputs)
ENTRIES = {
    "k256_mul_batch": (2 * 256, _k256),
    "x448": (3 * 128, _x448),
    "ed448_verify": (2 * 128, _ed448_verify),
    "ed448_mul_gen": (2 * 128, _ed448_mul_gen),
}


@pytest.mark.parametrize("entry", list(ENTRIES))
def test_two_shards_on_one_device(entry):
    import ecgpu

    per_sm, make = ENTRIES[entry]
    n, wave = _sizes(per_sm)
    first, run, refuse = make(n)
    one, two = ecgpu.Engine([0]), ecgpu.Engine([0, 0])
    try:
        for e in (one, two):
            e.timing_enable(True)
        want = run(one, first)
        got = run(two, first)
        assert np.array_equal(got, want)
        for e in (one, two):
            ms, calls = e.timing_read()
            assert calls == 1 and ms > 0
        if refuse is not None:
            # the second shard starts at n / 2: refused records in its second and third chunks, the first one reported
            bad = first.copy()
            at = n // 2 + wave + 7
            refuse(bad, at)
            refuse(bad, at + wave)
            for e in (one, two):
                with pytest.raises(ecgpu.EcgError) as ei:
                    run(e, bad)
                assert ei.value.code == ecgpu.ECG_ESCALAR_RANGE and ei.value.index == at
            assert np.array_equal(run(two, first), want)  # the ctx is usable after a refused call
    finally:
        one.close()
        two.close()
