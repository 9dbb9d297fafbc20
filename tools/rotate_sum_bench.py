"""Sums of rotations on one GPU: sb200_apply_galois_add and sb200_rotate_sum against the device chain they replace
(sb200_apply_galois into a temporary, then a two-operand sb200_add_many into the accumulator, per step), run alternately on the
same seeded inputs with the outputs compared word for word.  Time from CUDA events around each call sequence (median of --reps),
the bytes the chain moves beyond the fused calls (per step and ciphertext: add_many reads two slabs of 2 polynomials and writes
one, the fused epilogue reads the addend's 2: 4 polynomials of L n words), and the card name and power limit read in the same run.
One JSON line per shape:
  - apply_galois_add and rotate_sum with count = 16 (4 keys of 3.6 GB each beside the batch): CKKS n = 65536, 32 primes, L = 31;
  - a full slot sum (rotate_sum over n / 2 slots, 13 steps): CKKS n = 16384, 8 primes, L = 7.
  python tools/rotate_sum_bench.py [--reps 5] [--batch 2]"""
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


def run_shape(S, torch, n, k, count, B, reps, what):
    L = k - 1
    mods = S.coeff_modulus_create(n, [50] * k)
    ctx = S.Context(S.CKKS, n, mods)
    rng = np.random.default_rng(7)
    hkey = np.stack([np.stack([np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(k)]) for _ in range(2)])
                     for _ in range(L)])
    steps = [1 << j for j in range(count.bit_length() - 1)]
    elts = [ctx.galois_elt_from_step(s) for s in steps]
    keys = [ctx.load_key(hkey) for _ in steps]  # one key's words under every element: the timing does not depend on them
    del hkey
    q = torch.tensor([int(m) for m in mods[:L]], dtype=torch.int64, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(1234 + n + count)
    x = torch.remainder(torch.randint(0, 1 << 62, (B, 2, L, n), dtype=torch.int64, device="cuda", generator=gen), q.view(1, 1, L, 1)).contiguous()
    a = torch.remainder(torch.randint(0, 1 << 62, (B, 2, L, n), dtype=torch.int64, device="cuda", generator=gen), q.view(1, 1, L, 1)).contiguous()
    y_f, y_c, t = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)

    if what == "apply_galois_add":
        def fused():
            ctx.d_apply_galois_add(x, elts[0], keys[0], a, y_f, L, B)

        def chain():
            ctx.d_apply_galois(x, elts[0], keys[0], t, L, B)
            ctx.d_add_many([a, t], y_c, L, B, [2, 2])
        nsteps = 1
    else:
        def fused():
            ctx.d_rotate_sum(x, elts, keys, y_f, L, B)

        def chain():
            y_c.copy_(x)
            for e, kk in zip(elts, keys):
                ctx.d_apply_galois(y_c, e, kk, t, L, B)
                ctx.d_add_many([y_c, t], y_c, L, B, [2, 2])
        nsteps = len(steps)

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
    extra = 4 * 8 * L * n * B * nsteps
    name, power = card()
    t_f, t_c = float(np.median(tf)), float(np.median(tc))
    return {"card": name, "power_limit": power, "op": what, "n": n, "L": L, "count": count if what == "rotate_sum" else None,
            "steps": nsteps, "batch": B, "fused_ms": round(t_f, 3), "chain_ms": round(t_c, 3), "speedup": round(t_c / t_f, 3),
            "fused_ms_all": [round(v, 3) for v in tf], "chain_ms_all": [round(v, 3) for v in tc],
            "chain_extra_bytes": extra, "outputs_equal": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=2, help="ciphertexts per call")
    args = ap.parse_args()
    import torch

    import seal_b200 as S

    for n, k, count, B, what in ((65536, 32, 2, args.batch, "apply_galois_add"), (65536, 32, 16, args.batch, "rotate_sum"),
                                 (16384, 8, 8192, 4 * args.batch, "rotate_sum")):
        print(json.dumps(run_shape(S, torch, n, k, count, B, args.reps, what)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
