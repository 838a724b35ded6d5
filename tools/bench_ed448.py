#!/usr/bin/env python3
"""Ed448 verification throughput of ecg_ed448_verify_batch on one GPU; prints one JSON line.

    python tools/bench_ed448.py [--n 1048576] [--steps 10] [--warmup 3]

The workload: n OpenSSL-made Ed448 signatures over 64-byte messages from 1,024 keys; one in 16 has a flipped message bit
(it runs the whole verification and is refused at the final comparison).
- verify_per_s: device-resident operands (ECG_FLAG_DEVICE_PTRS), n signatures per step, CUDA events around each step;
- host_verify_per_s: the same signatures from and to host buffers (chunk pipeline, copies included), host clock;
- kernel_ms: the verification kernel's own time per step (ecg_timing_read);
- imad_peak / imad_fraction: the IMAD.WIDE rate of ecg_microbench(0) in the same run, and the share of it that the
  algorithmic multiplier count (IMAD_PER_VERIFY below) reaches at the kernel's rate;
- bit_exact: every verdict of the last timed step (and of the host-buffer run) against OpenSSL on all host cores, and
  the first `model_checked` of them against the Python model (tests/ed448_model.py), outside the timed regions;
- cpu_baseline_verify_per_s: OpenSSL's Ed448 verification on the same host cores.
There is no CPU fallback: without a CUDA device the script fails."""
import argparse
import json
import multiprocessing as mp
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "elliptic-curves_b200"), os.path.join(ROOT, "tests")]

# multiplier slots (IMAD.WIDE) per verification, from ecg_ed448.cuh: M = mulNxN<14> (196), S = sqrN<14> (105), a
# multiplication by a small constant 14.  Two decompressions with the subgroup test (1,359 S + 43 M + 5 small each), the
# -A table (1 M, one doubling, 7 additions of 9 M, 9 small), 444 doublings (3 M + 4 S, + 1 M for T before the 159 that
# precede an addition), 112 additions of 9 M (-A) and 64 of 8 M (B), the final comparison (2 M), and the six folds of
# the wide reduction mod ell (17 x 7 each).  SHAKE256 runs on the ALU and is not counted.
M14, S14, SMALL = 14 * 14, 14 * 15 // 2, 14
IMAD_PER_VERIFY = (2 * (1359 * S14 + 43 * M14 + 5 * SMALL) + (M14 + 4 * M14 + 4 * S14 + 7 * 9 * M14 + 9 * SMALL)
                   + 444 * (3 * M14 + 4 * S14) + 159 * M14 + 112 * 9 * M14 + 64 * 8 * M14 + 2 * M14 + 6 * 17 * 7)
MSG_LEN, KEYS = 64, 1024


def _sign_chunk(args):
    seeds, msgs = args
    from cryptography.hazmat.primitives.asymmetric.ed448 import Ed448PrivateKey

    keys = [Ed448PrivateKey.from_private_bytes(s) for s in seeds]
    pks = [k.public_key().public_bytes_raw() for k in keys]
    return [(pks[i % len(keys)], keys[i % len(keys)].sign(m)) for i, m in enumerate(msgs)]


def _verify_chunk(args):
    from cryptography.exceptions import InvalidSignature
    from cryptography.hazmat.primitives.asymmetric.ed448 import Ed448PublicKey

    out = bytearray()
    for pk, sig, msg in zip(*args):
        try:
            Ed448PublicKey.from_public_bytes(pk).verify(sig, msg)
            out.append(1)
        except (InvalidSignature, ValueError):
            out.append(0)
    return bytes(out)


def _chunks(n, procs):
    step = (n + procs * 8 - 1) // (procs * 8)
    return [(i, min(n, i + step)) for i in range(0, n, step)]


def openssl_verify_many(PK, SG, MS, procs):
    n = len(PK) // 57
    jobs = [([PK[57 * i:57 * i + 57] for i in range(a, b)], [SG[114 * i:114 * i + 114] for i in range(a, b)],
             [MS[MSG_LEN * i:MSG_LEN * i + MSG_LEN] for i in range(a, b)]) for a, b in _chunks(n, procs)]
    with mp.Pool(procs) as pool:
        return np.frombuffer(b"".join(pool.map(_verify_chunk, jobs)), np.uint8)


def workload(n, procs):
    rng = np.random.default_rng(448)
    seeds = [bytes(rng.integers(0, 256, 57, dtype=np.uint8)) for _ in range(KEYS)]
    MS = rng.integers(0, 256, MSG_LEN * n, dtype=np.uint8)
    msgs = [MS[MSG_LEN * i:MSG_LEN * i + MSG_LEN].tobytes() for i in range(n)]
    # chunks aligned to KEYS, so that signature i is made with key i % KEYS
    step = max(KEYS, ((n + procs * 4 - 1) // (procs * 4) + KEYS - 1) // KEYS * KEYS)
    with mp.Pool(procs) as pool:
        parts = pool.map(_sign_chunk, [(seeds, msgs[a:a + step]) for a in range(0, n, step)])
    pairs = [p for part in parts for p in part]
    PK = np.frombuffer(b"".join(p for p, _ in pairs), np.uint8).copy()
    SG = np.frombuffer(b"".join(s for _, s in pairs), np.uint8).copy()
    MS[MSG_LEN * np.arange(7, n, 16)] ^= 1  # one in 16: the signed message no longer matches
    return PK, SG, MS


def gpu_info():
    import subprocess

    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": q[0], "power_limit_w": float(q[1]), "sm_max_mhz": float(q[2])}
    except Exception:  # noqa: BLE001 - the name still comes from torch
        import torch

        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_max_mhz": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--model-checked", type=int, default=256)
    a = ap.parse_args()
    import torch

    import ecgpu

    if not torch.cuda.is_available():
        sys.exit("bench_ed448: no CUDA device (there is no CPU fallback)")
    n, procs = a.n, os.cpu_count() or 1
    PK, SG, MS = workload(n, procs)
    offs = np.arange(n + 1, dtype=np.uint64) * MSG_LEN
    rec = {"metric": "ed448_verify_per_s", "n": n, "msg_len": MSG_LEN, "steps": a.steps, "warmup": a.warmup, **gpu_info()}

    # device-resident operands
    eng = ecgpu.Engine([0], device_ptrs=True)
    pkd, sgd, msd = torch.from_numpy(PK).cuda(), torch.from_numpy(SG).cuda(), torch.from_numpy(MS).cuda()
    od = torch.from_numpy(offs.view(np.int64)).cuda()
    vd = torch.empty(n, dtype=torch.uint8, device="cuda")
    call = lambda: eng.ed448_verify_ptr(n, pkd.data_ptr(), sgd.data_ptr(), msd.data_ptr(), od.data_ptr(), vd.data_ptr())  # noqa: E731
    for _ in range(a.warmup):
        call()
    torch.cuda.synchronize()
    eng.timing_enable(True)
    times = []
    for _ in range(a.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()  # the call returns after its stream has drained
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    kms, kcalls = eng.timing_read()
    eng.timing_enable(False)
    step_ms = float(np.median(times))
    rec["verify_per_s"] = n / (step_ms * 1e-3)
    rec["step_ms_median"], rec["step_ms_min"], rec["step_ms_max"] = step_ms, min(times), max(times)
    rec["kernel_ms"] = kms / max(kcalls, 1)
    rec["kernel_verify_per_s"] = n / (rec["kernel_ms"] * 1e-3)
    v_last = vd.cpu().numpy().copy()

    peak, _ = eng.microbench(0)
    rec["imad_per_verify"] = IMAD_PER_VERIFY
    rec["imad_peak_per_s"] = peak
    rec["imad_fraction"] = rec["kernel_verify_per_s"] * IMAD_PER_VERIFY / peak
    eng.close()

    # host buffers: chunk pipeline, copies included
    heng = ecgpu.Engine([0])
    v_h = np.empty(n, np.uint8)
    heng.ed448_verify_packed(PK, SG, MS, offs, valid=v_h)
    t = []
    for _ in range(max(3, a.steps // 3)):
        t0 = time.perf_counter()
        heng.ed448_verify_packed(PK, SG, MS, offs, valid=v_h)
        t.append(time.perf_counter() - t0)
    rec["host_verify_per_s"] = n / float(np.median(t))
    heng.close()

    # correctness, outside the timed regions
    PKb, SGb, MSb = PK.tobytes(), SG.tobytes(), MS.tobytes()
    ref = openssl_verify_many(PKb, SGb, MSb, procs)
    import ed448_model

    m = min(n, a.model_checked)
    model = [int(ed448_model.verify(PKb[57 * i:57 * i + 57], SGb[114 * i:114 * i + 114], MSb[MSG_LEN * i:MSG_LEN * i + MSG_LEN]))
             for i in range(m)]
    rec["bit_exact"] = bool(np.array_equal(v_last, ref) and np.array_equal(v_h, ref) and list(v_last[:m]) == model)
    rec["verdicts_checked_openssl"], rec["verdicts_checked_model"] = n, m
    rec["valid_fraction"] = float(v_last.mean())

    # the CPU baseline: OpenSSL Ed448 verification on all host cores
    mb = min(n, 1 << 16)
    t0 = time.perf_counter()
    openssl_verify_many(PKb[:57 * mb], SGb[:114 * mb], MSb[:MSG_LEN * mb], procs)
    rec["cpu_baseline_verify_per_s"] = mb / (time.perf_counter() - t0)
    rec["cpu_cores"] = procs
    rec["speedup_vs_cpu"] = rec["verify_per_s"] / rec["cpu_baseline_verify_per_s"]
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
