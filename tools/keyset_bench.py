#!/usr/bin/env python
"""tools/keyset_bench.py -- loading key streams onto the device in one pass (sb200_kswitch_keys_load) against one
sb200_kswitch_key_load call per key, which parses the object again (and inflates it again, for zlib) for every key.

    python tools/keyset_bench.py [--reps 2] [--no-cpp]

Shapes:
  * BFV n = 16384, 8 primes of 54 bits, the default Galois set (GaloisTool::get_elts_all): the seeded stream KeyGenerator's
    Serializable overloads save (written by the device's generator) and the reference's GaloisKeys::save(compr_mode zlib) of the same
    set (oracle/_ref/libsealref_keyset.so);
  * CKKS n = 65536, 32 primes of 30 bits, a seeded stream of two Galois keys (each handle holds 3.6 GB).
Each time is the best of --reps, with every handle freed before the next run; the timed region ends in a device synchronise, and
is measured with CUDA events on the default stream and with the host clock.  Then, unless --no-cpp, the C++ batch load of 64 seeded
ciphertexts at n = 32768 against seal::Ciphertext::load plus Evaluator::upload (oracle/_ref/bin/shim_keyset_test --bench).  Prints
the card's name and power limit, one line per measurement and one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        return "unknown"


def timed(fn, reps):
    """best (event ms, host ms) of reps calls of fn; fn returns the handles it made, freed before the next call"""
    import torch

    best = (float("inf"), float("inf"))
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record()
        keys = fn()
        e1.record()
        torch.cuda.synchronize()
        host = (time.perf_counter() - t0) * 1e3
        best = min(best, (e0.elapsed_time(e1), host), key=lambda x: x[1])
        del keys
    return best


def compare(label, ctx, stream, slots, reps, out):
    one = timed(lambda: ctx.load_kswitch_keys(stream, slots), reps)
    loop = timed(lambda: [ctx.load_key_stream(stream, s) for s in slots], reps)
    print(f"{label}: {len(slots)} keys, {len(stream) / 2 ** 20:.0f} MiB stream: one pass {one[0]:.1f} ms (host {one[1]:.1f}), "
          f"one call per key {loop[0]:.1f} ms (host {loop[1]:.1f}), x{loop[1] / one[1]:.2f}")
    out[label] = {"keys": len(slots), "stream_bytes": len(stream), "one_pass_ms": one[0], "one_pass_host_ms": one[1],
                  "per_key_ms": loop[0], "per_key_host_ms": loop[1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--no-cpp", action="store_true")
    a = ap.parse_args()
    import oracle as O
    import refseal as R
    import seal_b200 as S
    from test_gpu_keyset_load import Ref, ZLIB

    gpu = card()
    print(f"card: {gpu}")
    out = {"card": gpu}
    rng = np.random.default_rng(1)
    # BFV n = 16384, 8 primes: the default Galois set
    n, mods = 16384, O.coeff_modulus_create(16384, [54] * 8)
    t = R.plain_modulus_batching(n, 20)
    r = Ref(S.BFV, n, mods, t)
    ctx = S.Context(S.BFV, n, mods, t)
    elts = r.elts_all()
    slots = sorted({(e - 1) // 2 for e in elts})  # get_elts_all lists n + 1 twice
    skd = ctx.load_secret_key(r.secret_key())
    seeded = ctx.generate_kswitch_keys_seeded(skd, elts)
    compare("bfv16384_default_set_seeded", ctx, seeded, slots, a.reps, out)
    zlib = r.galois_keys(None, ZLIB)
    compare("bfv16384_default_set_zlib", ctx, zlib, slots, a.reps, out)
    del ctx, skd
    # CKKS n = 65536, 32 primes: two Galois keys
    n, mods = 65536, O.coeff_modulus_create(65536, [30] * 32)
    ctx = S.Context(S.CKKS, n, mods)
    skd = ctx.load_secret_key(np.stack([rng.integers(0, q, n, dtype=np.uint64) for q in mods]))
    elts = [ctx.galois_elt_from_step(1), ctx.galois_elt_from_step(2)]
    stream = ctx.generate_kswitch_keys_seeded(skd, elts)
    compare("ckks65536_two_keys_seeded", ctx, stream, sorted((e - 1) // 2 for e in elts), a.reps, out)
    del ctx, skd
    shim = os.path.join(ROOT, "oracle", "_ref", "bin", "shim_keyset_test")
    if not a.no_cpp and os.path.exists(shim):
        line = subprocess.run([shim, "--bench"], capture_output=True, text=True, check=True).stdout.strip()
        print(line)
        out["cpp_batch_load"] = line
    print(json.dumps(out))


if __name__ == "__main__":
    main()
