"""Write bandwidth of the scalar CKKS encoder (sb200_ckks_encode_scalar, real kind) on one GPU: B plaintexts of L primes at degree n,
each a constant polynomial written by ckks_fill_kernel (B L n 8 bytes, nothing read but B values).
  - call: CUDA events around whole stream calls (the B values' D2H copy and the stream synchronisation included), median of --reps;
  - kernel: the fill kernel's own device time from the library's profile (sb200_profile_read), in a separate pass.
Both as GB/s written against the H100 SXM data sheet's 3.35 TB/s of HBM3 bandwidth.  Prints one JSON line with the card name and
its power limit, read in the same run.
  python tools/ckks_scalar_bw.py [--n 65536] [--primes 32] [--batch 64] [--reps 20]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM data sheet, HBM3


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
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch

    import seal_b200 as S

    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing measured")
    n, L, B = args.n, args.primes, args.batch
    mods = S.coeff_modulus_create(n, [50] * L)
    ctx = S.Context(S.CKKS, n, mods)
    values = torch.from_numpy(np.linspace(-100.0, 100.0, B)).cuda()
    plain = torch.empty((B, L, n), dtype=torch.int64, device="cuda")
    scale = 2.0 ** 40
    written = 8.0 * B * L * n

    def call():
        ctx.d_ckks_encode_scalar(values, plain, L, B, S.Context.CKKS_SCALAR_REAL, scale)

    for _ in range(3):  # warm-up: module load, first launches
        call()
    torch.cuda.synchronize()
    ts = []
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    call_ms = float(np.median(ts))

    ctx.profile(True)
    for _ in range(args.reps):
        call()
    torch.cuda.synchronize()
    rows = {name: (ms, launches) for name, ms, launches, _ in ctx.profile_read()}
    ctx.profile(False)
    fill_ms_total, launches = rows["ckks_fill"]
    fill_ms = fill_ms_total / launches

    # the plaintexts are the constant polynomials: spot-check one member against the host entry point
    want = ctx.ckks_encode_scalar(np.array([values[B // 2].item()]), L, scale)
    assert (plain[B // 2].cpu().numpy().view(np.uint64) == want[0]).all(), "device plaintext differs from the host entry point"

    name, power = card()
    print(json.dumps({
        "op": "sb200_ckks_encode_scalar (real)", "n": n, "primes": L, "batch": B, "bytes_written": written,
        "call_ms": round(call_ms, 4), "call_GBps": round(written / call_ms / 1e6, 1),
        "fill_kernel_ms": round(fill_ms, 4), "fill_kernel_GBps": round(written / fill_ms / 1e6, 1),
        "fill_kernel_share_of_3.35TBps": round(written / fill_ms * 1e3 / PEAK_BYTES_PER_S, 3),
        "gpu": name, "power_limit": power,
    }))


if __name__ == "__main__":
    main()
