#!/usr/bin/env python3
"""Decaf448 throughput of ecg_decaf448_mul_batch (k P), ecg_decaf448_mul_gen_batch (k G), ecg_decaf448_lincomb and
ecg_decaf448_hash_to_curve_batch (RO) on one GPU; prints one JSON line.

    python tools/bench_decaf448.py [--n-mul 1048576] [--n-gen 4194304] [--n-lin 1048576] [--n-h2c 4194304] [--steps 5] [--warmup 2]

The workload: random secret scalars a < ell and their elements [a]G (1,024 of them as the points of k P and of the linear
combination), random scalars k < ell, and 32-byte random messages under the suite's RO DST.
Per entry (mul, mul_gen, lincomb, h2c):
- <entry>_per_s: device-resident operands (ECG_FLAG_DEVICE_PTRS), CUDA events around each step (median);
- <entry>_host_per_s: the same from and to host buffers (chunk pipeline, copies included), host clock;
- <entry>_kernel_ms: the dominant kernel's own time per step (ecg_timing_read);
- <entry>_imad_fraction: the algorithmic IMAD.WIDE count below at the kernel's rate, against ecg_microbench(0) in the
  same run;
- <entry>_bit_exact: mul_gen: every output of the last step against the model's encode of [(-2k) mod ell]B computed by
  ecg_ed448_mul_gen_batch on a sample, and every output against the variable-base path on G; mul: every output against
  mul_gen(k a mod ell) and a sample against the model; lincomb: against mul_gen(sum k_i a_i mod ell) and the model's sum
  over the first terms; h2c: a sample against the model.
There is no CPU fallback: without a CUDA device the script fails."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "elliptic-curves_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

# multiplier slots (IMAD.WIDE) per element, from ecg_decaf448.cuh and ecg_ed448_group.cuh: M = mulNxN<14> (196),
# S = sqrN<14> (105), a multiplication by a small constant 14.
#   inverse square root a^((p - 3) / 4): 451 S + 12 M; decode: one of them and its check (1 S + 1 M) + 3 S + 10 M + 1 small;
#   encode: one of them + 1 S + 8 M + 2 small;
#   variable base and fixed base: as in bench_ed448_group.py;
#   map: one inverse square root + its check, 3 S + 10 M + 3 small; twisted addition 9 M + 1 small; twisted compress: one
#   inverse square root + 1 S + 7 M + 2 small; RO hash: two maps, one addition, one compress (Keccak runs on the ALU pipe).
M14, S14, SMALL = 14 * 14, 14 * 15 // 2, 14
ISR = 451 * S14 + 12 * M14
DECODE = ISR + 4 * S14 + 11 * M14 + SMALL
ENCODE = ISR + S14 + 8 * M14 + 2 * SMALL
VARBASE = (M14 + 4 * M14 + 4 * S14 + 7 * 9 * M14 + 9 * SMALL) + 444 * (3 * M14 + 4 * S14) + 111 * M14 + 112 * 9 * M14
FIXED = 56 * 8 * M14
MAP = ISR + 4 * S14 + 11 * M14 + 3 * SMALL
H2C = 2 * MAP + (9 * M14 + SMALL) + (ISR + S14 + 7 * M14 + 2 * SMALL)
IMAD = {"mul": DECODE + VARBASE, "mul_gen": FIXED, "lincomb": DECODE + VARBASE, "h2c": H2C}
L = 2**446 - 13818066809895115352007386748515426880336692474882178609894547503885
NPOINTS = 1024
DST = b"decaf448_XOF:SHAKE256_D448MAP_RO_"


def enc(ks, width=56):
    return np.frombuffer(b"".join(k.to_bytes(width, "little") for k in ks), np.uint8).copy()


def time_device(eng, call, steps, warmup):
    import torch

    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    eng.timing_enable(True)
    times = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()  # the call returns after its stream has drained
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    kms, kcalls = eng.timing_read()
    eng.timing_enable(False)
    return float(np.median(times)), kms / max(kcalls, 1)


def time_host(call, steps):
    call()
    t = []
    for _ in range(max(3, steps)):
        t0 = time.perf_counter()
        call()
        t.append(time.perf_counter() - t0)
    return float(np.median(t))


def rows(a):
    return [bytes(r) for r in np.asarray(a, np.uint8).reshape(-1, 56)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-mul", type=int, default=1 << 20)
    ap.add_argument("--n-gen", type=int, default=1 << 22)
    ap.add_argument("--n-lin", type=int, default=1 << 20)
    ap.add_argument("--n-h2c", type=int, default=1 << 22)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--model-checked", type=int, default=256)
    a = ap.parse_args()
    import torch

    import decaf448_model as D
    import ecgpu
    import ed448_model as M
    from bench_ed448 import gpu_info

    if not torch.cuda.is_available():
        sys.exit("bench_decaf448: no CUDA device (there is no CPU fallback)")
    rec = {"metric": "decaf448_per_s", "n_mul": a.n_mul, "n_gen": a.n_gen, "n_lin": a.n_lin, "n_h2c": a.n_h2c, "steps": a.steps,
           "warmup": a.warmup, **gpu_info()}
    rng = np.random.default_rng(448)
    ngen, nmax = a.n_gen, max(a.n_mul, a.n_lin)
    gks = [int.from_bytes(rng.bytes(56), "little") % L for _ in range(ngen)]
    ks = [int.from_bytes(rng.bytes(56), "little") % L for _ in range(nmax)]
    secrets = [int.from_bytes(rng.bytes(56), "little") % L for _ in range(NPOINTS)]
    GK, K = enc(gks), enc(ks)
    heng = ecgpu.Engine([0])
    pubs = heng.decaf448_mul_gen(enc(secrets)).reshape(-1).tobytes()
    PT = np.frombuffer(pubs * ((nmax + NPOINTS - 1) // NPOINTS), np.uint8)[:56 * nmax].copy()
    pt_secret = [secrets[i % NPOINTS] for i in range(nmax)]
    msgs = np.frombuffer(rng.bytes(32 * a.n_h2c), np.uint8).copy()
    offs = np.arange(0, 32 * a.n_h2c + 1, 32, dtype=np.uint64)

    eng = ecgpu.Engine([0], device_ptrs=True)
    peak, _ = eng.microbench(0)
    rec["imad_peak_per_s"] = peak
    out = {}
    gd, god = torch.from_numpy(GK).cuda(), torch.empty(56 * ngen, dtype=torch.uint8, device="cuda")
    ms, kms = time_device(eng, lambda: eng.decaf448_mul_gen_ptr(ngen, gd.data_ptr(), god.data_ptr()), a.steps, a.warmup)
    out["mul_gen"] = (ngen, ms, kms, god.cpu().numpy())
    del gd, god
    n = a.n_mul
    kd, pd, od = torch.from_numpy(K[:56 * n]).cuda(), torch.from_numpy(PT[:56 * n]).cuda(), torch.empty(56 * n, dtype=torch.uint8, device="cuda")
    ms, kms = time_device(eng, lambda: eng.decaf448_mul_ptr(n, kd.data_ptr(), pd.data_ptr(), od.data_ptr()), a.steps, a.warmup)
    out["mul"] = (n, ms, kms, od.cpu().numpy())
    del kd, pd, od
    n = a.n_lin
    kd, pd, od = torch.from_numpy(K[:56 * n]).cuda(), torch.from_numpy(PT[:56 * n]).cuda(), torch.empty(56, dtype=torch.uint8, device="cuda")
    ms, kms = time_device(eng, lambda: eng.decaf448_lincomb_ptr(n, kd.data_ptr(), pd.data_ptr(), od.data_ptr()), a.steps, a.warmup)
    out["lincomb"] = (n, ms, kms, od.cpu().numpy())
    del kd, pd, od
    n = a.n_h2c
    md, mo, hd = torch.from_numpy(msgs).cuda(), torch.from_numpy(offs.view(np.int64)).cuda(), torch.empty(56 * n, dtype=torch.uint8, device="cuda")
    ms, kms = time_device(eng, lambda: eng.decaf448_hash_to_curve_ptr(n, md.data_ptr(), mo.data_ptr(), hd.data_ptr(), DST), a.steps, a.warmup)
    out["h2c"] = (n, ms, kms, hd.cpu().numpy())
    del md, mo, hd
    for name, (n, ms, kms, _) in out.items():
        rec[f"{name}_per_s"] = n / (ms * 1e-3)
        rec[f"{name}_step_ms"] = ms
        rec[f"{name}_kernel_ms"] = kms
        rec[f"{name}_imad_per_elem"] = IMAD[name]
        rec[f"{name}_imad_fraction"] = n / (kms * 1e-3) * IMAD[name] / peak
    eng.close()

    # host buffers: chunk pipeline, copies included
    og = np.empty(56 * ngen, np.uint8)
    rec["mul_gen_host_per_s"] = ngen / time_host(lambda: heng.decaf448_mul_gen(GK, out=og), max(1, a.steps // 2))
    om = np.empty(56 * a.n_mul, np.uint8)
    rec["mul_host_per_s"] = a.n_mul / time_host(lambda: heng.decaf448_mul(K[:56 * a.n_mul], PT[:56 * a.n_mul], out=om), max(1, a.steps // 2))
    ol = []
    rec["lincomb_host_per_s"] = a.n_lin / time_host(lambda: ol.append(heng.decaf448_lincomb(K[:56 * a.n_lin], PT[:56 * a.n_lin])), max(1, a.steps // 2))
    oh = []
    rec["h2c_host_per_s"] = a.n_h2c / time_host(lambda: oh.append(heng.decaf448_hash_to_curve_packed(msgs, offs, DST)), max(1, a.steps // 2))

    # correctness, outside the timed regions
    m = a.model_checked
    g_last = out["mul_gen"][3]
    ed = heng.ed448_mul_gen(enc([D.gen_scalar(k) for k in gks[:m]], 57))
    ed_ok = all(D.encode(M.decompress_unchecked(bytes(ed[i]))) == bytes(g_last[56 * i:56 * i + 56]) for i in range(m))
    var = heng.decaf448_mul(GK, np.frombuffer(D.GENERATOR_BYTES * ngen, np.uint8)).reshape(-1)
    rec["mul_gen_bit_exact"] = bool(ed_ok and np.array_equal(g_last, og) and np.array_equal(g_last, var))
    n = a.n_mul
    want = heng.decaf448_mul_gen(enc([k * s % L for k, s in zip(ks[:n], pt_secret[:n])])).reshape(-1)
    model_ok = all(bytes(out["mul"][3][56 * i:56 * i + 56]) == D.mul(enc([ks[i]]).tobytes(), pubs[56 * (i % NPOINTS):56 * (i % NPOINTS) + 56])
                   for i in range(min(n, m)))
    rec["mul_bit_exact"] = bool(np.array_equal(out["mul"][3], want) and np.array_equal(om, want) and model_ok)
    n = a.n_lin
    want = bytes(heng.decaf448_mul_gen(enc([sum(k * s for k, s in zip(ks[:n], pt_secret[:n])) % L]))[0])
    mm = min(n, m)
    part = bytes(heng.decaf448_lincomb(K[:56 * mm], PT[:56 * mm]))
    model_part = D.lincomb([enc([k]).tobytes() for k in ks[:mm]], [pubs[56 * (i % NPOINTS):56 * (i % NPOINTS) + 56] for i in range(mm)])
    rec["lincomb_bit_exact"] = bool(bytes(out["lincomb"][3]) == want and all(bytes(o) == want for o in ol) and part == model_part)
    h_last = rows(out["h2c"][3])
    step = max(1, a.n_h2c // (4 * m))
    h_ok = all(h_last[i] == D.hash_to_curve(msgs[32 * i:32 * i + 32].tobytes(), DST) for i in range(0, a.n_h2c, step))
    rec["h2c_bit_exact"] = bool(h_ok and all(np.array_equal(o.reshape(-1), out["h2c"][3]) for o in oh))
    rec["bit_exact"] = rec["mul_gen_bit_exact"] and rec["mul_bit_exact"] and rec["lincomb_bit_exact"] and rec["h2c_bit_exact"]
    rec["model_checked"] = m
    heng.close()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
