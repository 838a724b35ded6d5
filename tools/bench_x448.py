#!/usr/bin/env python3
"""X448 throughput of ecg_x448_batch on one GPU; prints one JSON line.

    python tools/bench_x448.py [--n 1048576] [--steps 10] [--warmup 3] [--variants]

- x448_per_s: device-resident operands (ECG_FLAG_DEVICE_PTRS), n pairs per step, CUDA events around each step;
- host_x448_per_s: the same pairs from and to host buffers (chunk pipeline, copies included), host clock;
- kernel_ms: the ladder kernel's own time per step (ecg_timing_read);
- imad_peak / imad_fraction: the IMAD.WIDE rate of ecg_microbench(0) in the same run, and the share of it that the
  algorithmic multiplier count (IMAD_PER_X448 below) reaches at the kernel's rate;
- bit_exact: every output of the last timed step against OpenSSL's X448 on all host cores (outside the timed region);
- cpu_baseline_x448_per_s: OpenSSL's X448 on the same host cores;
- --variants: also the kernel time of both field variants (inlined / call-based) under the production launch bound,
  from the device test library, alternated in the same process.
There is no CPU fallback: without a CUDA device the script fails."""
import argparse
import ctypes
import json
import multiprocessing as mp
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "elliptic-curves_b200"), os.path.join(ROOT, "tests")]

# multiplier slots (IMAD.WIDE) per X448: 448 ladder steps of 5 M (196 each: mulNxN<14>) + 4 S (105: sqrN<14>) + one
# mul_small (14), the inversion chain (453 S + 13 M), the final U * W^-1 (1 M).  The reductions use no multiplier.
M14, S14, SMALL = 14 * 14, 14 * 15 // 2, 14
IMAD_PER_X448 = 448 * (5 * M14 + 4 * S14 + SMALL) + (453 * S14 + 13 * M14) + M14


def _openssl_chunk(args):
    ks, us = args
    from cryptography.hazmat.primitives.asymmetric.x448 import X448PrivateKey, X448PublicKey

    out = []
    for k, u in zip(ks, us):
        try:
            out.append(X448PrivateKey.from_private_bytes(k).exchange(X448PublicKey.from_public_bytes(u)))
        except ValueError:  # OpenSSL refuses an all-zero result
            out.append(bytes(56))
    return b"".join(out)


def openssl_many(K, U, procs):
    n = len(K) // 56
    recs_k = [K[56 * i:56 * i + 56] for i in range(n)]
    recs_u = [U[56 * i:56 * i + 56] for i in range(n)]
    step = (n + procs * 8 - 1) // (procs * 8)
    jobs = [(recs_k[i:i + step], recs_u[i:i + step]) for i in range(0, n, step)]
    with mp.Pool(procs) as pool:
        return b"".join(pool.map(_openssl_chunk, jobs))


def gpu_info():
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
    ap.add_argument("--variants", action="store_true")
    a = ap.parse_args()
    import torch

    import ecgpu

    if not torch.cuda.is_available():
        sys.exit("bench_x448: no CUDA device (there is no CPU fallback)")
    n, procs = a.n, os.cpu_count() or 1
    rng = np.random.default_rng(448)
    K = rng.integers(0, 256, 56 * n, dtype=np.uint8)
    U = rng.integers(0, 256, 56 * n, dtype=np.uint8)
    rec = {"metric": "x448_per_s", "n": n, "steps": a.steps, "warmup": a.warmup, **gpu_info()}

    # device-resident operands
    eng = ecgpu.Engine([0], device_ptrs=True)
    kd, ud = torch.from_numpy(K).cuda(), torch.from_numpy(U).cuda()
    od, okd = torch.empty(56 * n, dtype=torch.uint8, device="cuda"), torch.empty(n, dtype=torch.uint8, device="cuda")
    call = lambda: eng.x448_ptr(n, kd.data_ptr(), ud.data_ptr(), od.data_ptr(), okd.data_ptr())  # noqa: E731
    for _ in range(a.warmup):
        call()
    torch.cuda.synchronize()
    eng.timing_enable(True)
    times = []
    for _ in range(a.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()  # the call returns after its stream has drained (the ctx's own stream, after e0 on the current one)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    kms, kcalls = eng.timing_read()
    eng.timing_enable(False)
    step_ms = float(np.median(times))
    rec["x448_per_s"] = n / (step_ms * 1e-3)
    rec["step_ms_median"], rec["step_ms_min"], rec["step_ms_max"] = step_ms, min(times), max(times)
    rec["kernel_ms"] = kms / max(kcalls, 1)
    rec["kernel_x448_per_s"] = n / (rec["kernel_ms"] * 1e-3)
    out_last = od.cpu().numpy().tobytes()
    ok_last = okd.cpu().numpy()

    # the IMAD.WIDE peak in the same run, and the share of it the algorithmic count reaches at the kernel's rate
    peak, _ = eng.microbench(0)
    rec["imad_per_x448"] = IMAD_PER_X448
    rec["imad_peak_per_s"] = peak
    rec["imad_fraction"] = rec["kernel_x448_per_s"] * IMAD_PER_X448 / peak
    eng.close()

    # host buffers: chunk pipeline, both copies included
    heng = ecgpu.Engine([0])
    out_h = np.empty(56 * n, np.uint8)
    ok_h = np.empty(n, np.uint8)
    heng.x448(K, U, out_h, ok_h)
    t = []
    for _ in range(max(3, a.steps // 3)):
        t0 = time.perf_counter()
        heng.x448(K, U, out_h, ok_h)
        t.append(time.perf_counter() - t0)
    rec["host_x448_per_s"] = n / float(np.median(t))
    heng.close()

    # correctness of the last timed step, outside the timed regions
    ref = openssl_many(K.tobytes(), U.tobytes(), procs)
    rec["bit_exact"] = bool(out_last == ref and out_h.tobytes() == ref and ok_last.all())
    rec["outputs_checked"] = n

    # the CPU baseline: OpenSSL X448 on all host cores
    m = min(n, 1 << 17)
    t0 = time.perf_counter()
    openssl_many(K[:56 * m].tobytes(), U[:56 * m].tobytes(), procs)
    rec["cpu_baseline_x448_per_s"] = m / (time.perf_counter() - t0)
    rec["cpu_cores"] = procs
    rec["speedup_vs_cpu"] = rec["x448_per_s"] / rec["cpu_baseline_x448_per_s"]

    if a.variants:
        lib = ctypes.CDLL(os.path.join(ROOT, "tests", "dev", "libecgx448dev.so"))
        u8p = ctypes.POINTER(ctypes.c_uint8)
        lib.dev_x448_time.argtypes = [ctypes.c_int, ctypes.c_size_t, u8p, u8p, u8p, ctypes.c_int, ctypes.POINTER(ctypes.c_float)]
        vo = np.empty(56 * n, np.uint8)
        ms = {0: [], 1: []}
        for rep in range(4):
            for v in (0, 1) if rep % 2 == 0 else (1, 0):
                f = ctypes.c_float(0)
                rc = lib.dev_x448_time(v, n, K.ctypes.data_as(u8p), U.ctypes.data_as(u8p), vo.ctypes.data_as(u8p), 3, ctypes.byref(f))
                assert rc == 0, rc
                assert vo.tobytes() == ref, f"variant {v}: outputs differ from OpenSSL"
                ms[v].append(f.value)
        rec["variant_kernel_ms"] = {"inlined": float(np.median(ms[0])), "call_based": float(np.median(ms[1]))}
        rec["shipped_variant"] = "call_based" if ctypes.CDLL(os.path.join(ROOT, "tests", "dev", "libecgx448dev.so")).dev_x448_shipped_variant() else "inlined"
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
