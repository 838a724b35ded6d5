#!/usr/bin/env python3
"""Ed448 group-operation throughput of ecg_ed448_mul_batch (k P), ecg_ed448_mul_gen_batch (k B) and ecg_ed448_lincomb,
and of hashing with ecg_ed448_hash_to_curve_batch (RO, NU) and ecg_ed448_hash_to_scalar_batch, on one GPU; prints one
JSON line.

    python tools/bench_ed448_group.py [--n-mul 1048576] [--n-gen 4194304] [--n-lin 1048576] [--n-hash 4194304]
                                      [--steps 5] [--warmup 2] [--hash-only]

The workload: secret scalars a(s) = clamp(SHAKE256(s)[:57]) mod ell of random seeds s, with OpenSSL's public keys
pub(s) = [a(s)]B, 1,024 of them as the points of k P and of the linear combination; random scalars k < ell.
Per entry (mul, mul_gen, lincomb):
- <entry>_per_s: device-resident operands (ECG_FLAG_DEVICE_PTRS), CUDA events around each step (median);
- <entry>_host_per_s: the same from and to host buffers (chunk pipeline, copies included), host clock;
- <entry>_kernel_ms: the scalar-multiplication kernel's own time per step (ecg_timing_read);
- <entry>_imad_fraction: the algorithmic IMAD.WIDE count below at the kernel's rate, against ecg_microbench(0) in the
  same run;
- <entry>_bit_exact: mul_gen: every output of the last step against OpenSSL's public keys; mul: every output of the
  last step against mul_gen(k a(s) mod ell) (the identity [k]([a]B) = [k a]B) and a sample against the Python model;
  lincomb: against mul_gen(sum k_i a_i mod ell) and the model's sum over the first terms.
Per hashing entry (h2c_ro, h2c_nu, h2s): 32-byte random messages, device-resident (messages, offsets and records), one
DST; <entry>_per_s end to end (the hash kernel and, for points, the normalisation kernel), <entry>_kernel_ms the hash
kernel alone, <entry>_imad_fraction its cost-model count at its rate against ecg_microbench(0), <entry>_bit_exact a
sample of the last step against the Python model (tests/ed448_h2c_model.py).  --hash-only runs these alone.
CPU baselines on the host cores: OpenSSL Ed448 key generation (a k B per key) and OpenSSL X448 (the same-size ladder on
the isogenous Montgomery curve) for the variable base.  There is no CPU fallback: without a CUDA device the script fails."""
import argparse
import json
import multiprocessing as mp
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "elliptic-curves_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

# multiplier slots (IMAD.WIDE) per element, from ecg_ed448_group.cuh: M = mulNxN<14> (196), S = sqrN<14> (105), a
# multiplication by a small constant 14.
#   decompression with the subgroup test: 1,359 S + 43 M + 5 small (as in bench_ed448.py);
#   variable base: the table (1 M, a doubling of 4 M + 4 S, 7 additions of 9 M, 9 small), 444 doublings (3 M + 4 S, and
#   1 M for T before each of the 111 that precede an addition), 112 additions of 9 M;
#   fixed base: 56 mixed additions of 8 M;
#   normalisation: 5 M per element and one inversion (453 S + 13 M) per slice of 32;
#   lincomb: a variable-base product per term, and one addition of 9 M + 1 small per term in the tree.
M14, S14, SMALL = 14 * 14, 14 * 15 // 2, 14
DECOMP = 1359 * S14 + 43 * M14 + 5 * SMALL
VARBASE = (M14 + 4 * M14 + 4 * S14 + 7 * 9 * M14 + 9 * SMALL) + 444 * (3 * M14 + 4 * S14) + 111 * M14 + 112 * 9 * M14
FIXED = 56 * 8 * M14
NORM = 5 * M14 + (453 * S14 + 13 * M14) // 32
IMAD = {"mul": DECOMP + VARBASE + NORM, "mul_gen": FIXED + NORM, "lincomb": DECOMP + VARBASE + 9 * M14 + SMALL}
# hashing (ecg_ed448_h2c.cuh; estimates from the code, not measurements; Keccak runs on the ALU pipe and is not counted):
#   the inverse-square-root chain (p - 3) / 4: 451 S + 12 M;
#   one map with the homogenised isogeny: the chain + 18 M + 8 S + 7 small;
#   RO kernel: two maps, one addition (9 M + 1 small), two doublings (3 M + 4 S, then 4 M + 4 S); NU kernel: one map and
#   the doublings; both then pay the normalisation's share NORM;
#   hash to scalar: the 6 folds of 17 x 7 products of the 114-byte reduction mod ell.
ISR = 451 * S14 + 12 * M14
MAP = ISR + 18 * M14 + 8 * S14 + 7 * SMALL
DBL2 = 7 * M14 + 8 * S14
H2C_KERNEL = {"h2c_ro": 2 * MAP + 9 * M14 + SMALL + DBL2, "h2c_nu": MAP + DBL2, "h2s": 6 * 17 * 7}
IMAD.update({"h2c_ro": H2C_KERNEL["h2c_ro"] + NORM, "h2c_nu": H2C_KERNEL["h2c_nu"] + NORM, "h2s": H2C_KERNEL["h2s"]})
H2C_DST = b"edwards448_XOF:SHAKE256_ELL2_RO_"
L = 2**446 - 13818066809895115352007386748515426880336692474882178609894547503885
NPOINTS = 1024


def _secret_chunk(seeds):
    import ed448_group_model as G

    return [G.secret_scalar(s) for s in seeds]


def _public_chunk(seeds):
    from cryptography.hazmat.primitives.asymmetric.ed448 import Ed448PrivateKey

    return b"".join(Ed448PrivateKey.from_private_bytes(s).public_key().public_bytes_raw() for s in seeds)


def _pieces(xs, procs):
    step = max(1, (len(xs) + procs * 8 - 1) // (procs * 8))
    return [xs[i:i + step] for i in range(0, len(xs), step)]


def _x448_chunk(n):
    from cryptography.hazmat.primitives.asymmetric.x448 import X448PrivateKey

    k, peer = X448PrivateKey.generate(), X448PrivateKey.generate().public_key()
    t0 = time.perf_counter()
    for _ in range(n):
        k.exchange(peer)
    return time.perf_counter() - t0


def _keygen_chunk(n):
    from cryptography.hazmat.primitives.asymmetric.ed448 import Ed448PrivateKey

    seeds = [os.urandom(57) for _ in range(n)]
    t0 = time.perf_counter()
    for s in seeds:
        Ed448PrivateKey.from_private_bytes(s).public_key()
    return time.perf_counter() - t0


def cpu_rate(fn, per_proc, procs):
    t0 = time.perf_counter()
    with mp.Pool(procs) as pool:
        pool.map(fn, [per_proc] * procs)
    return per_proc * procs / (time.perf_counter() - t0)


def enc(ks):
    return np.frombuffer(b"".join(k.to_bytes(57, "little") for k in ks), np.uint8).copy()


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


def bench_hash(a):
    """the hashing entries on n 32-byte messages, device-resident end to end"""
    import torch

    import ecgpu
    import ed448_h2c_model as H

    n = a.n_hash
    rng = np.random.default_rng(9380)
    data = rng.integers(0, 256, 32 * n, dtype=np.uint8)
    offs = np.arange(0, 32 * (n + 1), 32, dtype=np.uint64)
    eng = ecgpu.Engine([0], device_ptrs=True)
    peak, _ = eng.microbench(0)
    rec = {"n_hash": n, "hash_msg_bytes": 32, "hash_imad_peak_per_s": peak}
    dd, do = torch.from_numpy(data).cuda(), torch.from_numpy(offs.view(np.int64)).cuda()
    od = torch.empty(57 * n, dtype=torch.uint8, device="cuda")
    calls = {"h2c_ro": lambda: eng.ed448_hash_to_curve_ptr(n, dd.data_ptr(), do.data_ptr(), od.data_ptr(), H2C_DST, False),
             "h2c_nu": lambda: eng.ed448_hash_to_curve_ptr(n, dd.data_ptr(), do.data_ptr(), od.data_ptr(), H2C_DST, True),
             "h2s": lambda: eng.ed448_hash_to_scalar_ptr(n, dd.data_ptr(), do.data_ptr(), od.data_ptr(), H2C_DST)}
    models = {"h2c_ro": lambda m: H.hash_to_curve(m, H2C_DST), "h2c_nu": lambda m: H.hash_to_curve(m, H2C_DST, True),
              "h2s": lambda m: H.hash_to_scalar(m, H2C_DST)}
    ok_all = True
    for name, call in calls.items():
        ms, kms = time_device(eng, call, a.steps, a.warmup)
        got = od.cpu().numpy()
        idx = sorted(set(np.linspace(0, n - 1, min(n, a.model_checked)).astype(int).tolist()))
        ok = all(bytes(got[57 * i:57 * i + 57]) == models[name](bytes(data[32 * i:32 * i + 32])) for i in idx)
        ok_all = ok_all and ok
        rec[f"{name}_per_s"] = n / (ms * 1e-3)
        rec[f"{name}_step_ms"] = ms
        rec[f"{name}_kernel_ms"] = kms
        rec[f"{name}_imad_per_elem"] = IMAD[name]
        rec[f"{name}_kernel_imad_per_elem"] = H2C_KERNEL[name]
        rec[f"{name}_imad_fraction"] = n / (kms * 1e-3) * H2C_KERNEL[name] / peak
        rec[f"{name}_bit_exact"] = ok
    rec["hash_model_checked"] = len(idx)
    rec["hash_bit_exact"] = ok_all
    eng.close()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-mul", type=int, default=1 << 20)
    ap.add_argument("--n-gen", type=int, default=1 << 22)
    ap.add_argument("--n-lin", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--model-checked", type=int, default=256)
    ap.add_argument("--n-hash", type=int, default=1 << 22)
    ap.add_argument("--hash-only", action="store_true")
    a = ap.parse_args()
    import torch

    import ecgpu
    import ed448_group_model as G
    import ed448_model as M
    from bench_ed448 import gpu_info

    if not torch.cuda.is_available():
        sys.exit("bench_ed448_group: no CUDA device (there is no CPU fallback)")
    if a.hash_only:
        rec = {"metric": "ed448_hash_per_s", "steps": a.steps, "warmup": a.warmup, **gpu_info()}
        rec.update(bench_hash(a))
        print(json.dumps(rec))
        return
    procs = os.cpu_count() or 1
    rng = np.random.default_rng(448)
    ngen = a.n_gen
    blob = rng.bytes(57 * ngen)
    seeds = [blob[57 * i:57 * i + 57] for i in range(ngen)]
    with mp.Pool(procs) as pool:
        secrets = [v for part in pool.map(_secret_chunk, _pieces(seeds, procs)) for v in part]
        pubs = b"".join(pool.map(_public_chunk, _pieces(seeds, procs)))
    rec = {"metric": "ed448_group_per_s", "n_mul": a.n_mul, "n_gen": ngen, "n_lin": a.n_lin, "steps": a.steps, "warmup": a.warmup,
           **gpu_info()}
    pyr = np.random.default_rng(57)
    nmax = max(a.n_mul, a.n_lin)
    ks = [int.from_bytes(pyr.bytes(56), "little") % L for _ in range(nmax)]
    K, A = enc(ks), enc(secrets)
    PT = np.frombuffer(pubs[:57 * NPOINTS] * ((nmax + NPOINTS - 1) // NPOINTS), np.uint8)[:57 * nmax].copy()
    pt_secret = [secrets[i % NPOINTS] for i in range(nmax)]

    eng = ecgpu.Engine([0], device_ptrs=True)
    peak, _ = eng.microbench(0)
    rec["imad_peak_per_s"] = peak
    out = {}
    # k B: device-resident
    ad, gd = torch.from_numpy(A).cuda(), torch.empty(57 * ngen, dtype=torch.uint8, device="cuda")
    ms, kms = time_device(eng, lambda: eng.ed448_mul_gen_ptr(ngen, ad.data_ptr(), gd.data_ptr()), a.steps, a.warmup)
    out["mul_gen"] = (ngen, ms, kms, gd.cpu().numpy())
    del ad, gd
    # k P
    n = a.n_mul
    kd, pd, od = torch.from_numpy(K[:57 * n]).cuda(), torch.from_numpy(PT[:57 * n]).cuda(), torch.empty(57 * n, dtype=torch.uint8, device="cuda")
    ms, kms = time_device(eng, lambda: eng.ed448_mul_ptr(n, kd.data_ptr(), pd.data_ptr(), od.data_ptr()), a.steps, a.warmup)
    out["mul"] = (n, ms, kms, od.cpu().numpy())
    del kd, pd, od
    # lincomb
    n = a.n_lin
    kd, pd, od = torch.from_numpy(K[:57 * n]).cuda(), torch.from_numpy(PT[:57 * n]).cuda(), torch.empty(57, dtype=torch.uint8, device="cuda")
    ms, kms = time_device(eng, lambda: eng.ed448_lincomb_ptr(n, kd.data_ptr(), pd.data_ptr(), od.data_ptr()), a.steps, a.warmup)
    out["lincomb"] = (n, ms, kms, od.cpu().numpy())
    del kd, pd, od
    for name, (n, ms, kms, _) in out.items():
        rec[f"{name}_per_s"] = n / (ms * 1e-3)
        rec[f"{name}_step_ms"] = ms
        rec[f"{name}_kernel_ms"] = kms
        rec[f"{name}_imad_per_elem"] = IMAD[name]
        rec[f"{name}_imad_fraction"] = n / (kms * 1e-3) * IMAD[name] / peak
    eng.close()

    # host buffers: chunk pipeline, copies included
    heng = ecgpu.Engine([0])
    og = np.empty(57 * ngen, np.uint8)
    rec["mul_gen_host_per_s"] = ngen / time_host(lambda: heng.ed448_mul_gen(A, out=og), max(1, a.steps // 2))
    om = np.empty(57 * a.n_mul, np.uint8)
    rec["mul_host_per_s"] = a.n_mul / time_host(lambda: heng.ed448_mul(K[:57 * a.n_mul], PT[:57 * a.n_mul], out=om), max(1, a.steps // 2))
    ol = []
    rec["lincomb_host_per_s"] = a.n_lin / time_host(lambda: ol.append(heng.ed448_lincomb(K[:57 * a.n_lin], PT[:57 * a.n_lin])), max(1, a.steps // 2))

    # correctness, outside the timed regions
    g_last = out["mul_gen"][3]
    pub_arr = np.frombuffer(pubs, np.uint8)
    rec["mul_gen_bit_exact"] = bool(np.array_equal(g_last, pub_arr) and np.array_equal(og, pub_arr))
    n = a.n_mul
    want = heng.ed448_mul_gen(enc([k * s % L for k, s in zip(ks[:n], pt_secret[:n])])).reshape(-1)
    m = min(n, a.model_checked)
    model_ok = all(bytes(out["mul"][3][57 * i:57 * i + 57]) == G.mul(G.enc_scalar(ks[i]), pubs[57 * (i % NPOINTS):57 * (i % NPOINTS) + 57])
                   for i in range(m))
    rec["mul_bit_exact"] = bool(np.array_equal(out["mul"][3], want) and np.array_equal(om, want) and model_ok)
    n = a.n_lin
    want = bytes(heng.ed448_mul_gen(enc([sum(k * s for k, s in zip(ks[:n], pt_secret[:n])) % L]))[0])
    mm = min(n, a.model_checked)
    part = bytes(heng.ed448_lincomb(K[:57 * mm], PT[:57 * mm]))
    model_part = G.lincomb([G.enc_scalar(k) for k in ks[:mm]], [pubs[57 * (i % NPOINTS):57 * (i % NPOINTS) + 57] for i in range(mm)])
    rec["lincomb_bit_exact"] = bool(bytes(out["lincomb"][3]) == want and all(bytes(o) == want for o in ol) and part == model_part)
    rec["bit_exact"] = rec["mul_gen_bit_exact"] and rec["mul_bit_exact"] and rec["lincomb_bit_exact"]
    rec["model_checked"] = m
    heng.close()
    assert M.encode(M.B) == M.B_BYTES

    # CPU baselines on the host cores
    rec["cpu_cores"] = procs
    rec["cpu_baseline_openssl_ed448_keygen_per_s"] = cpu_rate(_keygen_chunk, 2000, procs)
    rec["cpu_baseline_openssl_x448_per_s"] = cpu_rate(_x448_chunk, 2000, procs)
    rec["speedup_mul_gen_vs_openssl_keygen"] = rec["mul_gen_per_s"] / rec["cpu_baseline_openssl_ed448_keygen_per_s"]
    rec["speedup_mul_vs_openssl_x448"] = rec["mul_per_s"] / rec["cpu_baseline_openssl_x448_per_s"]
    rec.update(bench_hash(a))
    rec["bit_exact"] = rec["bit_exact"] and rec["hash_bit_exact"]
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
