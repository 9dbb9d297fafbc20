#!/usr/bin/env python
"""tools/keygen_bench.py -- key generation on the device against the reference's KeyGenerator, from the same secret key.

    python tools/keygen_bench.py [--reps 3] [--ref-galois N]

Shapes: BFV n = 16384, 8 primes of 54 bits (bench.py's rotation sweep) and CKKS n = 65536, 32 primes of 55 bits (the headline).
Device (sb200_kswitch_key_generate), after a warm-up that makes every key of the shape once:
  * the relinearization key into a host buffer (best of --reps);
  * the default Galois set (GaloisTool::get_elts_all) into host buffers: one reused buffer, the keys made one after another;
  * the same set into device handles (the handle also holds the integer key-switching path's copy of the key); each handle is
    freed after it is timed, since the n = 65536 set does not fit in 80 GB at once.
Every device time is a host clock around calls that end in a device synchronise.  Reference: seal::KeyGenerator
(oracle/_ref/libsealref_keygen.so, one thread) for the relinearization key and the first --ref-galois elements of the default set
(default: all of them), per key.  Prints the card's name and power limit, one line per measurement and one JSON line.

    python tools/keygen_bench.py --stream [--reps 3] [--ref-galois N]

times the seed-compressed streams instead (what KeyGenerator's Serializable overloads save with compr_mode none): the relinearization
key (best of --reps) and the default Galois set in one call (sb200_kswitch_keys_generate_seeded) into a pageable host buffer, after a
warm-up call into the same buffer; next to them, in the same run, the host-words path above (relinearization key, Galois set) and
the reference's create_relin_keys().save / create_galois_keys(elts).save(none) (oracle/_ref/libsealref_serial.so, one thread, the
first --ref-galois elements one per call).  Device times are CUDA events on the default stream and a host clock around each call."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SHAPES = [("BFV", 1, 16384, [54] * 8), ("CKKS", 2, 65536, [55] * 32)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-galois", type=int, default=None, help="reference Galois keys to time per shape (default: the whole set)")
    ap.add_argument("--stream", action="store_true", help="time the seed-compressed key streams")
    args = ap.parse_args()
    if args.stream:
        return stream_main(args)

    import torch

    import keygen_ref as K
    import refseal as R
    import seal_b200 as S

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the device times need an H100")
    if not K.ref_available():
        raise SystemExit("oracle/_ref/libsealref_keygen.so is missing (oracle/keygen.mk)")
    print(f"card: {card()}", flush=True)
    lib, results = S.lib(), []
    for name, scheme, n, bits in SHAPES:
        mods = R.coeff_modulus_create(n, bits)
        t = R.plain_modulus_batching(n, 20) if scheme == S.BFV else 0
        k = len(mods)
        ref = K.RefKeygen(scheme, n, mods, t)
        elts = ref.galois_elts_all()
        ctx = S.Context(scheme, n, mods, t)
        skd = ctx.load_secret_key(ref.secret_key())
        buf = np.zeros((k - 1, 2, k, n), dtype=np.uint64)
        seeds = ref.boot_seeds(k - 1)

        def to_host(elt):
            S._check(lib.sb200_kswitch_key_generate(ctx.h, skd.h, elt, 1, 1, S._hp(seeds), S._hp(buf), None))

        def to_handle(elt):
            h = C.c_void_p()
            S._check(lib.sb200_kswitch_key_generate(ctx.h, skd.h, elt, 1, 1, S._hp(seeds), None, C.byref(h)))
            return h

        def timed(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            return time.perf_counter() - t0, out

        for elt in [0] + elts:  # warm-up: every key of the shape once, both outputs (also builds the Galois tables)
            to_host(elt)
            lib.sb200_kswitch_key_destroy(to_handle(elt))
        relin = min(timed(lambda: to_host(0))[0] for _ in range(args.reps))
        gal_host = sum(timed(lambda: to_host(e))[0] for e in elts)
        gal_dev = 0.0
        for e in elts:
            dt, h = timed(lambda: to_handle(e))
            gal_dev += dt
            lib.sb200_kswitch_key_destroy(h)
        ref_elts = elts if args.ref_galois is None else elts[:args.ref_galois]
        t0 = time.perf_counter()
        ref.kswitch_key(0, keep=False)
        ref_relin = time.perf_counter() - t0
        t0 = time.perf_counter()
        for e in ref_elts:
            ref.kswitch_key(e, keep=False)
        ref_gal = time.perf_counter() - t0
        gb = (k - 1) * 2 * k * n * 8 / 1e9
        r = {"shape": f"{name} n={n} k={k}", "galois_keys": len(elts), "key_gb": round(gb, 3),
             "device_relin_host_ms": round(relin * 1e3, 2), "device_galois_set_host_s": round(gal_host, 3),
             "device_galois_set_handles_s": round(gal_dev, 3), "device_galois_host_ms_per_key": round(gal_host / len(elts) * 1e3, 2),
             "ref_relin_ms": round(ref_relin * 1e3, 1), "ref_galois_keys_timed": len(ref_elts),
             "ref_galois_ms_per_key": round(ref_gal / max(len(ref_elts), 1) * 1e3, 1),
             "speedup_relin_host": round(ref_relin / relin, 1),
             "speedup_galois_host_per_key": round(ref_gal / max(len(ref_elts), 1) / (gal_host / len(elts)), 1)}
        print(f"{r['shape']}: relin key {r['device_relin_host_ms']} ms (device -> host) vs {r['ref_relin_ms']} ms (reference); "
              f"{len(elts)} Galois keys {r['device_galois_set_host_s']} s (host) / {r['device_galois_set_handles_s']} s (handles) vs "
              f"{r['ref_galois_ms_per_key']} ms per key (reference, {len(ref_elts)} keys)", flush=True)
        results.append(r)
        del ctx, skd, ref
    print(json.dumps({"card": card(), "results": results}))


def stream_main(args):
    import torch

    import refseal as R
    import seal_b200 as S
    import test_gpu_serializable as T

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the device times need an H100")
    if not os.path.exists(T._REF):
        raise SystemExit("oracle/_ref/libsealref_serial.so is missing (oracle/serial.mk)")
    print(f"card: {card()}", flush=True)
    lib, results = S.lib(), []

    def timed(fn):
        """(wall seconds, CUDA-event seconds) of fn, which ends in a device synchronise"""
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, a.elapsed_time(b) / 1e3

    for name, scheme, n, bits in SHAPES:
        mods = R.coeff_modulus_create(n, bits)
        t = R.plain_modulus_batching(n, 20) if scheme == S.BFV else 0
        k = len(mods)
        ref = T.Ref(scheme, n, mods, t, 1)
        elts = galois_elts_all(scheme, n, mods, t)
        ctx = S.Context(scheme, n, mods, t)
        skd = ctx.load_secret_key(ref.secret_key())
        words = np.zeros((k - 1, 2, k, n), dtype=np.uint64)
        seeds = ref.seeds(len(elts) * (k - 1))

        def stream(es):
            arr = (C.c_uint32 * len(es))(*es)
            size = lib.sb200_kswitch_keys_save_seeded_size(ctx.h, arr, len(es))
            out = np.empty(size, dtype=np.uint8)

            def call():
                S._check(lib.sb200_kswitch_keys_generate_seeded(ctx.h, skd.h, arr, len(es), 1, 1, S._hp(seeds), out.ctypes.data, size))
            return call, size

        relin_call, relin_bytes = stream([0])
        gal_call, gal_bytes = stream(elts)
        relin_call(), gal_call()  # warm-up: page the buffers in, build the Galois tables
        relin = min((timed(relin_call) for _ in range(args.reps)), key=lambda x: x[0])
        gal = timed(gal_call)
        del gal_call

        def to_host(elt):
            S._check(lib.sb200_kswitch_key_generate(ctx.h, skd.h, elt, 1, 1, S._hp(seeds), S._hp(words), None))

        to_host(0)
        words_relin = min(timed(lambda: to_host(0))[0] for _ in range(args.reps))
        words_gal = sum(timed(lambda: to_host(e))[0] for e in elts)
        ref_elts = elts if args.ref_galois is None else elts[:args.ref_galois]
        t0 = time.perf_counter()
        ref.relin_keys()
        ref_relin = time.perf_counter() - t0
        t0 = time.perf_counter()
        for e in ref_elts:
            ref.galois_keys([e])
        ref_gal = (time.perf_counter() - t0) / max(len(ref_elts), 1)
        r = {"shape": f"{name} n={n} k={k}", "galois_keys": len(elts),
             "relin_stream_gb": round(relin_bytes / 1e9, 3), "galois_stream_gb": round(gal_bytes / 1e9, 3),
             "stream_relin_ms": round(relin[0] * 1e3, 2), "stream_relin_event_ms": round(relin[1] * 1e3, 2),
             "stream_galois_set_s": round(gal[0], 3), "stream_galois_set_event_s": round(gal[1], 3),
             "stream_galois_gb_per_s": round(gal_bytes / 1e9 / gal[0], 2),
             "words_relin_ms": round(words_relin * 1e3, 2), "words_galois_set_s": round(words_gal, 3),
             "ref_relin_save_ms": round(ref_relin * 1e3, 1), "ref_galois_keys_timed": len(ref_elts),
             "ref_galois_save_ms_per_key": round(ref_gal * 1e3, 1)}
        print(f"{r['shape']}: seeded relin stream {r['stream_relin_ms']} ms ({r['relin_stream_gb']} GB) vs host words "
              f"{r['words_relin_ms']} ms vs reference {r['ref_relin_save_ms']} ms; {len(elts)} Galois keys as one stream "
              f"{r['stream_galois_set_s']} s ({r['galois_stream_gb']} GB, {r['stream_galois_gb_per_s']} GB/s) vs host words "
              f"{r['words_galois_set_s']} s vs reference {r['ref_galois_save_ms_per_key']} ms per key ({len(ref_elts)} keys)", flush=True)
        results.append(r)
        del ctx, skd, ref
    print(json.dumps({"card": card(), "mode": "stream", "results": results}))


def galois_elts_all(scheme, n, mods, t):
    """GaloisTool::get_elts_all() of the shape, from the reference"""
    import keygen_ref as K

    return K.RefKeygen(scheme, n, mods, t).galois_elts_all()


if __name__ == "__main__":
    main()
