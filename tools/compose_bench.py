"""Batch compositions on one GPU at n = 65536 with 32 primes:
  - device time of sb200_add_many over m operand batches against m - 1 chained sb200_add calls (CUDA events, median of --reps);
  - wall time of Evaluator::multiply_many and exponentiate(16) on CiphertextBatch against the same products made one
    multiply_relinearize_inplace call per pair in the reference's order (oracle/_ref/bin/shim_compose_test --bench).
Prints one JSON line per half, with the card name and its power limit.
  python tools/compose_bench.py [--m 16] [--batch 64] [--product-batch 16] [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        name, power = (v.strip() for v in q.stdout.splitlines()[0].split(","))
        return name, power
    except Exception:  # no nvidia-smi: the numbers still print
        import torch

        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=65536)
    ap.add_argument("--primes", type=int, default=32)
    ap.add_argument("--m", type=int, default=16)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--product-batch", type=int, default=16, help="batch of the multiply_many half (its staging is 3x the operands)")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch

    import seal_b200 as S

    n, k, m, B = args.n, args.primes, args.m, args.batch
    mods = S.coeff_modulus_create(n, [50] * k)
    ctx = S.Context(S.CKKS, n, mods)
    L, size = k, 2
    words = B * size * L * n
    ops = [torch.randint(0, 1 << 40, (words,), dtype=torch.int64, device="cuda") for _ in range(m)]
    out = torch.empty(words, dtype=torch.int64, device="cuda")

    def timed(f):
        ts = []
        for _ in range(args.reps + 1):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return float(np.median(ts[1:]))

    def fold():
        ctx.d_add_many(ops, out, L, B, [size] * m)

    def chained():
        lib = S.lib()
        st = ctx._stream()
        S._check(lib.sb200_add(ctx.h, L, size, B, S._dp(ops[0]), S._dp(ops[1]), S._dp(out), st))
        for j in range(2, m):
            S._check(lib.sb200_add(ctx.h, L, size, B, S._dp(out), S._dp(ops[j]), S._dp(out), st))

    def pair_fold():
        ctx.d_add_many(ops[:2], out, L, B, [size] * 2)

    def pair_add():
        S._check(S.lib().sb200_add(ctx.h, L, size, B, S._dp(ops[0]), S._dp(ops[1]), S._dp(out), ctx._stream()))

    name, power = card()
    slab_gb = words * 8 / 1e9
    t_fold, t_chain = timed(fold), timed(chained)
    t_pf, t_pa = timed(pair_fold), timed(pair_add)
    print(json.dumps({"card": name, "power_limit": power, "n": n, "primes": k, "operands": m, "batch": B,
                      "add_many_ms": round(t_fold, 3), "chained_add_ms": round(t_chain, 3),
                      "add_many_GBps": round((m + 1) * slab_gb / t_fold * 1e3, 1),
                      "chained_GBps": round(3 * (m - 1) * slab_gb / t_chain * 1e3, 1),
                      "pair_fold_ms": round(t_pf, 3), "pair_sb200_add_ms": round(t_pa, 3)}), flush=True)
    del ops, out
    torch.cuda.empty_cache()
    exe = os.path.join(ROOT, "oracle", "_ref", "bin", "shim_compose_test")
    if os.path.exists(exe):
        r = subprocess.run([exe, "--bench", str(n), str(k), str(m), str(args.product_batch)], capture_output=True, text=True)
        line = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else "{}"
        res = json.loads(line) if r.returncode == 0 else {"error": r.stderr[-400:]}
        res.update({"card": name, "power_limit": power})
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
