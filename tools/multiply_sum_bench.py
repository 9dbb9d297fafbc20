"""Sums of ciphertext products on one GPU: sb200_multiply_sum against the chain it replaces (sb200_multiply of every term into a
size-3 temporary, then one sb200_add_many over the K products), with and without one sb200_relinearize of each sum, run
alternately on the same seeded inputs with the outputs compared word for word.  Kernel time from CUDA events (median of --reps),
algorithmic bytes from the shapes, and the card name and power limit read in the same run; one JSON line per shape:
CKKS n = 65536, 32 primes at L = 31, K in {16, 64}, M in {1, 4}, B ciphertexts per operand (the chain's K intermediates
of every output must fit: 48.75 MB each per member at this shape).
  python tools/multiply_sum_bench.py [--reps 3] [--batch 2]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBPS = 3.35  # H100 SXM data sheet


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        name, power = (v.strip() for v in q.stdout.splitlines()[0].split(","))
        return name, power
    except Exception:  # no nvidia-smi: the numbers still print
        import torch

        return torch.cuda.get_device_name(0), "unknown"


def run_shape(S, torch, ctx, mods, key, n, L, K, M, B, reps):
    q = torch.tensor([int(m) for m in mods[:L]], dtype=torch.int64, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(1234 + K + M)

    def residues(shape):  # uniform words below each row's prime, [.., L, n]
        x = torch.randint(0, 1 << 62, shape, dtype=torch.int64, device="cuda", generator=gen)
        return torch.remainder(x, q.view(*([1] * (len(shape) - 2)), L, 1)).contiguous()

    lhs = [residues((B, 2, L, n)) for _ in range(M * K)]
    rhs = [residues((B, 2, L, n)) for _ in range(K)]
    outs = [torch.empty((B, 3, L, n), dtype=torch.int64, device="cuda") for _ in range(M)]
    ref = [torch.empty_like(o) for o in outs]
    outs2 = [torch.empty((B, 2, L, n), dtype=torch.int64, device="cuda") for _ in range(M)]
    ref2 = [torch.empty_like(o) for o in outs2]
    temps = [torch.empty((B, 3, L, n), dtype=torch.int64, device="cuda") for _ in range(K)]

    def fused(relin):
        ctx.d_multiply_sum(lhs, rhs, outs, L, B)
        if relin:
            for j in range(M):
                ctx.d_relinearize(outs[j], key, outs2[j], L, B)

    def chain(relin):  # the lazy-relinearization idiom: K products, add_many, then one relinearization per sum
        for j in range(M):
            for i in range(K):
                ctx.d_multiply(lhs[j * K + i], rhs[i], temps[i], L, B)
            ctx.d_add_many(temps, ref[j], L, B, [3] * K)
            if relin:
                ctx.d_relinearize(ref[j], key, ref2[j], L, B)

    def timed(f, relin):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        f(relin)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    res = {}
    for relin in (False, True):
        timed(fused, relin), timed(chain, relin)  # warm-up of both
        tf, tc = [], []
        for _ in range(reps):  # alternating
            tf.append(timed(fused, relin))
            tc.append(timed(chain, relin))
        same = all(torch.equal(a, b) for a, b in zip(outs, ref))
        if relin:
            same = same and all(torch.equal(a, b) for a, b in zip(outs2, ref2))
        res[relin] = (float(np.median(tf)), float(np.median(tc)), same)
    w = 8 * L * n * B  # bytes of one polynomial of every member
    tiles = -(-M // 2)  # output tiles of kMultiplySumTile = 2
    fused_bytes = w * (2 * K * tiles + 2 * M * K + 3 * M)
    chain_bytes = w * (M * K * (4 + 3) + M * (3 * K + 3))  # multiply: 4 reads, 3 writes per term; add_many: K reads of 3, 3 writes
    name, power = card()
    t_f, t_c, same = res[False]
    t_fr, t_cr, same_r = res[True]
    return {"card": name, "power_limit": power, "n": n, "L": L, "K": K, "M": M, "batch": B,
            "multiply_sum_ms": round(t_f, 3), "chain_ms": round(t_c, 3), "speedup": round(t_c / t_f, 2),
            "multiply_sum_bytes": fused_bytes, "chain_bytes": chain_bytes,
            "multiply_sum_TBps": round(fused_bytes / t_f / 1e9, 3), "multiply_sum_frac_of_3.35TBps": round(fused_bytes / t_f / 1e9 / HBM_TBPS, 3),
            "chain_TBps": round(chain_bytes / t_c / 1e9, 3),
            "with_relinearize": {"multiply_sum_ms": round(t_fr, 3), "chain_ms": round(t_cr, 3), "speedup": round(t_cr / t_fr, 2)},
            "outputs_equal": bool(same and same_r)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=2, help="ciphertexts per operand")
    args = ap.parse_args()
    import torch

    import seal_b200 as S

    n, k = 65536, 32
    L = k - 1
    mods = S.coeff_modulus_create(n, [50] * k)
    ctx = S.Context(S.CKKS, n, mods)
    rng = np.random.default_rng(7)
    key = ctx.load_key(np.stack([np.stack([np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(k)]) for _ in range(2)])
                                 for _ in range(L)]))
    for K in (16, 64):
        for M in (1, 4):
            print(json.dumps(run_shape(S, torch, ctx, mods, key, n, L, K, M, args.batch, args.reps)), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
