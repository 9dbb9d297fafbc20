"""Sums of plaintext products on one GPU: sb200_multiply_plain_sum against the chain it replaces (multiply_plain_n of every term into
a temporary, then add_many), run alternately on the same seeded inputs with the outputs compared word for word.  Kernel time from
CUDA events (median of --reps), algorithmic bytes from the shapes, and the card name and power limit; one JSON line per shape:
  - CKKS n = 65536, 32 primes, K = 16 ciphertexts, M = 1 and M = 8 outputs, shared plaintexts (a linear transform's giant step);
  - BFV n = 8192, 3 primes, K = 4096 shared NTT-form plaintexts, B = 16 queries, M = 1 (a PIR answer).
  python tools/plain_sum_bench.py [--reps 5] [--batch 4]"""
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


def run_shape(S, torch, label, scheme, n, k, K, M, B, reps, group=64):
    mods = S.coeff_modulus_create(n, [50] * k if scheme == S.CKKS else [60] * k)
    t = 0 if scheme == S.CKKS else 65537
    ctx = S.Context(scheme, n, mods, t)
    L, size = k, 2
    q = torch.tensor([int(m) for m in mods[:L]], dtype=torch.int64, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(1234)

    def residues(shape):  # uniform words below each row's prime, [.., L, n]
        x = torch.randint(0, 1 << 62, shape, dtype=torch.int64, device="cuda", generator=gen)
        return torch.remainder(x, q.view(*([1] * (len(shape) - 2)), L, 1)).contiguous()

    cts = [residues((B, size, L, n)) for _ in range(K)]
    plains = [residues((1, L, n)) for _ in range(M * K)]
    outs = [torch.empty((B, size, L, n), dtype=torch.int64, device="cuda") for _ in range(M)]
    ref = [torch.empty_like(o) for o in outs]
    g = min(group, K)
    temps = [torch.empty((B, size, L, n), dtype=torch.int64, device="cuda") for _ in range(g)]
    st = ctx._stream()
    lib = S.lib()

    def fused():
        ctx.d_multiply_plain_sum(cts, plains, outs, L, B, [size] * K, [1] * (M * K))

    def chain():  # multiply_plain_n of each term into a temporary; add_many over a group of terms (and the partial sum)
        for j in range(M):
            for i0 in range(0, K, g):
                i1 = min(K, i0 + g)
                for i in range(i0, i1):
                    S._check(lib.sb200_multiply_plain_n(ctx.h, L, size, B, 1, S._dp(cts[i]), S._dp(plains[j * K + i]), S._dp(temps[i - i0]), st))
                ops = ([ref[j]] if i0 else []) + temps[: i1 - i0]
                ctx.d_add_many(ops, ref[j], L, B, [size] * len(ops))

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        f()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    timed(fused), timed(chain)  # warm-up of both
    tf, tc = [], []
    for _ in range(reps):  # alternating
        tf.append(timed(fused))
        tc.append(timed(chain))
    same = all(torch.equal(a, b) for a, b in zip(outs, ref))
    w = 8 * L * n
    tiles = -(-M // 4) if M >= 3 else 1
    fused_bytes = w * (K * B * size * tiles + M * K + M * B * size)
    chain_bytes = w * (M * K * (2 * B * size + 1) + M * K * B * size + M * B * size + M * max(0, -(-K // g) - 1) * B * size)
    t_f, t_c = float(np.median(tf)), float(np.median(tc))
    name, power = card()
    return {"shape": label, "card": name, "power_limit": power, "n": n, "primes": k, "K": K, "M": M, "batch": B,
            "plain_sum_ms": round(t_f, 3), "chain_ms": round(t_c, 3), "speedup": round(t_c / t_f, 2),
            "plain_sum_GBps": round(fused_bytes / t_f / 1e6, 1), "plain_sum_frac_of_3.35TBps": round(fused_bytes / t_f / 1e9 / HBM_TBPS, 3),
            "chain_GBps": round(chain_bytes / t_c / 1e6, 1), "outputs_equal": bool(same)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=4, help="ciphertexts per term of the CKKS shapes")
    args = ap.parse_args()
    import torch

    import seal_b200 as S

    for label, scheme, n, k, K, M, B in (("ckks_giant_step_M1", S.CKKS, 65536, 32, 16, 1, args.batch),
                                         ("ckks_giant_step_M8", S.CKKS, 65536, 32, 16, 8, args.batch),
                                         ("bfv_pir", S.BFV, 8192, 3, 4096, 1, 16)):
        res = run_shape(S, torch, label, scheme, n, k, K, M, B, args.reps)
        print(json.dumps(res), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
