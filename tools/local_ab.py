#!/usr/bin/env python
"""tools/local_ab.py -- A/B of two builds of the library on bench.py's headline run, for changes to the integer key-switching
path's local passes: the library under test (seal_b200/libseal_b200.so as built) and a baseline build (--base, e.g. the parent
commit's library built into build/) are swapped into seal_b200/libseal_b200.so and run alternately, so both series see the same
card, clocks and neighbours.  The library under test is put back at the end.

    python tools/local_ab.py --base build/parent/libseal_b200.so [--pairs 3] [--steps 5] [--warmup 2]

Prints the card (name, power limit, max SM clock), one line per run (ciphertexts/s, verified.ok, ms per step of ks32_fwd_local and
ks32_inv_local) and a summary of the pairs as one JSON line."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "seal_b200", "libseal_b200.so")
KERNELS = ("ks32_fwd_local", "ks32_inv_local")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        return "unknown"


def run(label, lib, args):
    shutil.copyfile(lib, LIB)
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup),
           "--no-cpu-baseline", "--no-configs", "--no-e2e"]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stderr)
        raise SystemExit(f"bench.py failed with the {label} library")
    res = json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("{")][-1])
    kern = {k["name"]: k for k in res["roofline"]["kernels"]}
    r = {"lib": label, "ct_per_s": round(res["value"], 1), "verified_ok": bool(res["verified"] and res["verified"]["ok"])}
    for name in KERNELS:
        r[name + "_ms_per_step"] = round(kern[name]["ms"] / args.steps, 3) if name in kern else float("nan")
    r["local_ms_per_step"] = round(sum(r[name + "_ms_per_step"] for name in KERNELS), 3)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="baseline libseal_b200.so")
    ap.add_argument("--pairs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    print("card:", card(), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        new = os.path.join(tmp, "libseal_b200.so")
        shutil.copyfile(LIB, new)
        libs = {"base": os.path.abspath(args.base), "new": new}
        pairs = []
        try:
            for _ in range(args.pairs):
                pair = {}
                for label in ("base", "new"):
                    pair[label] = run(label, libs[label], args)
                    print(json.dumps(pair[label]), flush=True)
                pairs.append(pair)
        finally:
            shutil.copyfile(new, LIB)
    summary = {
        "card": card(),
        "ct_per_s": {m: [p[m]["ct_per_s"] for p in pairs] for m in ("base", "new")},
        "speedup_per_pair": [round(p["new"]["ct_per_s"] / p["base"]["ct_per_s"], 4) for p in pairs],
        "local_ms_saved_per_pair": [round(p["base"]["local_ms_per_step"] - p["new"]["local_ms_per_step"], 3) for p in pairs],
        "verified_ok": all(p[m]["verified_ok"] for p in pairs for m in ("base", "new")),
    }
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
