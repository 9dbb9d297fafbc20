"""Plaintext matrix times encrypted vector by diagonals on one GPU: sb200_diagonal_sum and sb200_apply_galois_multiply_plain_add
against the device chain they replace (per term: sb200_apply_galois into a temporary, sb200_multiply_plain_n on it, then a
two-operand sb200_add_many into the destination; the first term's product is the destination), run alternately on the same seeded
inputs with the outputs compared word for word.  Time from CUDA events around each call sequence (median of --reps), the bytes the
chain moves beyond the fused calls (per rotated term with an addend and per ciphertext: the product pass reads 2 + 1 polynomials
and writes 2, the add pass reads 4 and writes 2, the fused epilogue reads the plaintext's 1 and the addend's 2: 8 polynomials of
L n words), and the card name and power limit read in the same run.  One JSON line per shape:
  - diagonal_sum with an identity term and 2 or 3 rotated terms, and apply_galois_multiply_plain_add (keys of 3.6 GB each beside the
    batch): CKKS n = 65536, 32 primes, L = 31 (the integer key-switching path);
  - diagonal_sum with an identity term and 3 rotated terms: CKKS n = 16384, 8 primes, L = 7 (the 64-bit key-switching path).
  python tools/diagonal_sum_bench.py [--reps 5] [--batch 2]"""
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


def run_shape(S, torch, n, k, rotated, B, reps, what):
    L = k - 1
    mods = S.coeff_modulus_create(n, [50] * k)
    ctx = S.Context(S.CKKS, n, mods)
    rng = np.random.default_rng(7)
    hkey = np.stack([np.stack([np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(k)]) for _ in range(2)])
                     for _ in range(L)])
    steps = [0] + list(range(1, rotated + 1))
    elts = [1 if s == 0 else ctx.galois_elt_from_step(s) for s in steps]
    keys = [None] + [ctx.load_key(hkey) for _ in range(rotated)]  # one key's words under every element: the timing does not depend on them
    del hkey
    q = torch.tensor([int(m) for m in mods[:L]], dtype=torch.int64, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(1234 + n + rotated)

    def rand(*shape):
        return torch.remainder(torch.randint(0, 1 << 62, shape, dtype=torch.int64, device="cuda", generator=gen),
                               q.view(*([1] * (len(shape) - 2)), L, 1)).contiguous()

    x, a = rand(B, 2, L, n), rand(B, 2, L, n)
    # shared and per-member diagonals alternate
    plains = [rand(1 if i % 2 == 0 else B, L, n) for i in range(len(steps))]
    counts = [p.shape[0] for p in plains]
    y_f, y_c, t = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)

    if what == "apply_galois_multiply_plain_add":
        def fused():
            ctx.d_apply_galois_multiply_plain_add(x, elts[1], keys[1], plains[1], counts[1], a, y_f, L, B)

        def chain():
            ctx.d_apply_galois(x, elts[1], keys[1], t, L, B)
            ctx.d_multiply_plain_n(t, plains[1], t, L, 2, B, counts[1])
            ctx.d_add_many([a, t], y_c, L, B, [2, 2])
    else:
        def fused():
            ctx.d_diagonal_sum(x, elts, keys, plains, counts, y_f, L, B)

        def chain():
            ctx.d_multiply_plain_n(x, plains[0], y_c, L, 2, B, counts[0])
            for e, kk, p, c in zip(elts[1:], keys[1:], plains[1:], counts[1:]):
                ctx.d_apply_galois(x, e, kk, t, L, B)
                ctx.d_multiply_plain_n(t, p, t, L, 2, B, c)
                ctx.d_add_many([y_c, t], y_c, L, B, [2, 2])

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
    same = bool(torch.equal(y_f, y_c))
    extra = 8 * 8 * L * n * B * rotated
    name, power = card()
    t_f, t_c = float(np.median(tf)), float(np.median(tc))
    return {"card": name, "power_limit": power, "op": what, "n": n, "L": L, "rotated_terms": rotated,
            "identity_terms": 1 if what == "diagonal_sum" else 0, "batch": B, "fused_ms": round(t_f, 3), "chain_ms": round(t_c, 3),
            "speedup": round(t_c / t_f, 3), "fused_ms_all": [round(v, 3) for v in tf], "chain_ms_all": [round(v, 3) for v in tc],
            "chain_extra_bytes": extra, "outputs_equal": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=2, help="ciphertexts per call")
    args = ap.parse_args()
    import torch

    import seal_b200 as S

    for n, k, rotated, B, what in ((65536, 32, 1, args.batch, "apply_galois_multiply_plain_add"), (65536, 32, 2, args.batch, "diagonal_sum"),
                                   (65536, 32, 3, args.batch, "diagonal_sum"), (16384, 8, 3, 4 * args.batch, "diagonal_sum")):
        print(json.dumps(run_shape(S, torch, n, k, rotated, B, args.reps, what)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
