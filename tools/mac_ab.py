#!/usr/bin/env python
"""tools/mac_ab.py -- A/B of the integer key-switching path's product step in one build: bench.py's headline run alternately with
SB200_KS_MAC_MMA=0 (the integer-pipe kernels) and =1 (the INT8 tensor-core kernel), so both series see the same card, clocks and
neighbours.

    python tools/mac_ab.py [--pairs 3] [--steps 5] [--warmup 2]

Prints the card (name, power limit, max SM clock), one line per run (ciphertexts/s, the ks32_mac kernel's ms per step and its
share of the profiled step, verified.ok) and a summary of the pairs as one JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        return "unknown"


def run(mma, args):
    env = dict(os.environ, SB200_KS_MAC_MMA=str(mma))
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup),
           "--no-cpu-baseline", "--no-configs", "--no-e2e"]
    p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stderr)
        raise SystemExit(f"bench.py failed with SB200_KS_MAC_MMA={mma}")
    res = json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("{")][-1])
    kern = {k["name"]: k for k in res["roofline"]["kernels"]}
    mac = kern.get("ks32_mac", {"ms": float("nan"), "share": float("nan")})
    return {"mma": mma, "ct_per_s": round(res["value"], 1), "ks32_mac_ms_per_step": round(mac["ms"] / args.steps, 3),
            "ks32_mac_share": mac["share"], "verified_ok": res["verified"]["ok"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    print("card:", card(), flush=True)
    pairs = []
    for i in range(args.pairs):
        pair = {}
        for mma in (0, 1):
            r = run(mma, args)
            print(json.dumps(r), flush=True)
            pair[mma] = r
        pairs.append(pair)
    summary = {
        "card": card(),
        "ct_per_s": {"mma0": [p[0]["ct_per_s"] for p in pairs], "mma1": [p[1]["ct_per_s"] for p in pairs]},
        "speedup_per_pair": [round(p[1]["ct_per_s"] / p[0]["ct_per_s"], 4) for p in pairs],
        "ks32_mac_ms_per_step": {"mma0": [p[0]["ks32_mac_ms_per_step"] for p in pairs], "mma1": [p[1]["ks32_mac_ms_per_step"] for p in pairs]},
        "verified_ok": all(p[m]["verified_ok"] for p in pairs for m in (0, 1)),
    }
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
