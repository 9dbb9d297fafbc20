#!/usr/bin/env python
"""tools/bench_ops.py -- device-resident throughput of every hot-path operation at the BASELINE.json config shapes
(uniform-random ciphertexts, synthetic keys).  Not the contract benchmark (bench.py is)."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import seal_b200 as S  # noqa: E402

CONFIGS = [
    ("cfg1 BFV n=4096 k=3 (BFVDefault)", S.BFV, 4096, None, 1024),
    ("cfg2 CKKS n=8192 k=4 (54-bit)", S.CKKS, 8192, [54] * 4, 1024),
    ("cfg3 CKKS n=32768 k=16 (55/56-bit)", S.CKKS, 32768, [55] * 15 + [56], 256),
    ("cfg4 BFV n=16384 k=8 (54-bit)", S.BFV, 16384, [54] * 8, 512),
    ("cfg5 CKKS n=65536 k=32 (55-bit)", S.CKKS, 65536, [55] * 32, 128),
]
BFV_DEFAULT_4096 = [0xFFFFEE001, 0xFFFFC4001, 0x1FFFFE0001]


def rand_rows(mods, n, prefix, nprimes, g):
    t = torch.empty((*prefix, nprimes, n), dtype=torch.int64, device="cuda")
    for i in range(nprimes):
        t[..., i, :] = torch.randint(0, mods[i], (*prefix, n), generator=g, dtype=torch.int64, device="cuda")
    return t


def timeit(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    rows = []
    for name, scheme, n, bits, batch in CONFIGS:
        mods = BFV_DEFAULT_4096 if bits is None else S.coeff_modulus_create(n, bits)
        k, L = len(mods), len(mods) - 1
        t = 1032193 if scheme == S.BFV and n == 4096 else (786433 if scheme == S.BFV else 0)
        ctx = S.Context(scheme, n, mods, t)
        key = ctx.load_key(rand_rows(mods, n, (L, 2), k, g).cpu().numpy().view(np.uint64))
        a, b = rand_rows(mods, n, (batch, 2), L, g), rand_rows(mods, n, (batch, 2), L, g)
        o3 = torch.empty((batch, 3, L, n), dtype=torch.int64, device="cuda")
        o2 = torch.empty((batch, 2, L, n), dtype=torch.int64, device="cuda")
        om = torch.empty((batch, 2, max(L - 1, 1), n), dtype=torch.int64, device="cuda")
        res = {"config": name, "batch": batch}
        res["multiply"] = batch / timeit(lambda: ctx.d_multiply(a, b, o3, L, batch)) * 1e3
        res["relinearize"] = batch / timeit(lambda: ctx.d_relinearize(o3, key, o2, L, batch)) * 1e3
        res["multiply+relinearize"] = batch / timeit(lambda: ctx.d_multiply_relinearize(a, b, key, o2, L, batch)) * 1e3
        ms = timeit(lambda: ctx.d_multiply_plain(a, b, o2, L, 2, batch))  # b's first [batch][L][n] words serve as the plaintexts
        res["multiply_plain"] = batch / ms * 1e3
        res["multiply_plain_GBps"] = batch * 5 * L * n * 8 / (ms * 1e-3) / 1e9
        elt = ctx.galois_elt_from_step(1)
        res["rotate (1 step)"] = batch / timeit(lambda: ctx.d_apply_galois(a, elt, key, o2, L, batch)) * 1e3
        if L > 1:
            f = ctx.d_rescale_to_next if scheme == S.CKKS else ctx.d_mod_switch_to_next
            res["rescale/mod_switch"] = batch / timeit(lambda: f(a, om, L, batch)) * 1e3
        ms = timeit(lambda: (ctx.d_ntt_inverse(a, L, 2, batch), ctx.d_ntt_forward(a, L, 2, batch)))
        res["ct NTT+INTT"] = batch / ms * 1e3
        res["ntt_GBps"] = 2 * batch * 2 * L * 2 * n * 8 / (ms * 1e-3) / 1e9
        rows.append(res)
        print(json.dumps(res), flush=True)
        del ctx, key, a, b, o3, o2, om
        torch.cuda.empty_cache()
    return rows


PRNG_CONFIGS = [(c[0], c[1], c[2], c[3], 1024 if c[0][:4] == "cfg2" else 32) for c in CONFIGS if c[0][:4] in ("cfg2", "cfg5")]
PRNG_NAMES = {1: "blake2xb", 2: "shake256"}


def seeded_stream(full, seed, prng):
    """the seed-compressed form of a saved size-2 ciphertext (Serializable<Ciphertext>, ciphertext.cpp:325-352): c_0 only, then
    UniformRandomGeneratorInfo behind its own SEALHeader (prng_type, 64-byte seed)"""
    hdr, members, count = 16, 73, int.from_bytes(full[105:113], "little")
    c0_words = count // 2
    inner = (16 + 8 + 8 * c0_words).to_bytes(8, "little")
    body = full[hdr:hdr + members] + full[89:97] + inner + c0_words.to_bytes(8, "little") + full[113:113 + 8 * c0_words]
    info = full[:8] + (16 + 1 + 64).to_bytes(8, "little") + bytes([prng]) + seed.tobytes()
    head = full[:8] + (hdr + len(body) + len(info)).to_bytes(8, "little")
    return head + body + info


def prng_main():
    """per PRNG type at cfg2 / cfg5: seeded-load and encrypt_zero_symmetric ciphertexts/s, the PRNG stream kernels' algorithmic
    GB/s (profile entries of the stream launcher: bytes written over device ms) and the batch-1 seeded-load latency"""
    rows = []
    for name, scheme, n, bits, batch in PRNG_CONFIGS:
        mods = S.coeff_modulus_create(n, bits)
        k, L = len(mods), len(mods) - 1
        ctx = S.Context(scheme, n, mods)
        rng = np.random.default_rng(5)
        sk = ctx.load_secret_key(np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(k)]))
        out = torch.empty((batch, 2, L, n), dtype=torch.int64, device="cuda")
        for prng in (1, 2):
            res = {"config": name, "batch": batch, "prng": PRNG_NAMES[prng]}
            seeds = rng.integers(0, 2 ** 63, (batch, 8), dtype=np.uint64)
            ms = timeit(lambda: ctx.d_encrypt_zero_symmetric(sk, out, L, batch, seeds, bootstrap_prng=prng, ciphertext_prng=prng))
            res["encrypt_zero_symmetric"] = batch / ms * 1e3
            pub = ctx.d_encrypt_zero_symmetric(sk, out, L, batch, seeds, save_seed=True, want_public_seeds=True, bootstrap_prng=prng,
                                               ciphertext_prng=prng)
            full = ctx.d_save_ciphertexts(out, L, 2, batch, is_ntt_form=True)
            streams = [seeded_stream(f, pub[b], prng) for b, f in enumerate(full)]
            dst = torch.empty_like(out)
            ms = timeit(lambda: ctx.d_load_ciphertexts(streams, dst, L, 2))
            res["seeded load"] = batch / ms * 1e3
            torch.cuda.synchronize()
            assert torch.equal(dst, out), "seeded load must re-create the encryptions"
            ctx.profile(True)
            ctx.d_load_ciphertexts(streams, dst, L, 2)
            torch.cuda.synchronize()
            ent = [e for e in ctx.profile_read() if e[0] == ("seed_stream" if prng == 1 else "seed_stream:shake256")]
            ctx.profile(False)
            res["prng_stream_GBps"] = ent[0][3] / (ent[0][1] * 1e-3) / 1e9
            res["prng_stream_ms"] = ent[0][1]
            if name.startswith("cfg5"):
                one = dst[:1]
                res["seeded load batch-1 latency ms"] = timeit(lambda: ctx.d_load_ciphertexts(streams[:1], one, L, 2), reps=10)
            rows.append(res)
            print(json.dumps(res), flush=True)
        del ctx, sk, out
        torch.cuda.empty_cache()
    return rows


NOISE_CONFIGS = [("BFV n=8192 BFVDefault", 8192, 1024), ("BFV n=32768 BFVDefault (15 data primes)", 32768, 128)]


def noise_main():
    """invariant_noise_budget of device-resident batches of fresh BFV encryptions: budgets/s, the noise_norm kernel's share of the
    call (profile entries), and the reference's rate on one core on the same ciphertexts"""
    import time

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import noise_ref as N
    import refseal as R

    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit": os.popen(
        "nvidia-smi --query-gpu=power.limit --format=csv,noheader -i 0").read().strip()}), flush=True)
    rows = []
    for name, n, batch in NOISE_CONFIGS:
        mods = R.coeff_modulus_bfv_default(n)
        t = R.plain_modulus_batching(n, 20)
        L = len(mods) - 1
        rc = R.RefContext(R.BFV, n, mods, t)
        ctx = S.Context(S.BFV, n, mods, t)
        sk = ctx.load_secret_key(rc.secret_key())
        d = torch.empty((batch, 2, L, n), dtype=torch.int64, device="cuda")
        ctx.d_encrypt_zero_symmetric(sk, d, L, batch)
        out = torch.empty(batch, dtype=torch.int32, device="cuda")
        res = {"config": name, "batch": batch}
        ms = timeit(lambda: ctx.d_invariant_noise_budget(d, sk, out, L, 2, batch))
        res["noise budgets/s"] = batch / ms * 1e3
        ctx.profile(True)
        ctx.d_invariant_noise_budget(d, sk, out, L, 2, batch)
        torch.cuda.synchronize()
        ent = ctx.profile_read()
        ctx.profile(False)
        total = sum(e[1] for e in ent)
        res["noise_norm share of device time"] = sum(e[1] for e in ent if e[0] == "noise_norm") / total
        host = d[:8].cpu().numpy().view(np.uint64)
        N.ref_budget(rc, L, host[0], False)  # the reference's context and Decryptor are built on first use: not timed
        t0 = time.perf_counter()
        ref = [N.ref_budget(rc, L, c, False) for c in host]
        res["reference 1-core budgets/s"] = len(host) / (time.perf_counter() - t0)
        assert [r[1] for r in ref] == [int(x) for x in out[:8].cpu()], "device and reference budgets differ"
        rows.append(res)
        print(json.dumps(res), flush=True)
        del ctx, sk, d, out
        torch.cuda.empty_cache()
    return rows


PLAIN_BATCH = 512


def alternate(fns, rounds=3, reps=5):
    """median ms per call of each of fns, timed in rounds that alternate between them (CUDA events, warm-up in timeit)"""
    times = [[] for _ in fns]
    for _ in range(rounds):
        for i, f in enumerate(fns):
            times[i].append(timeit(f, reps))
    return [sorted(t)[len(t) // 2] for t in times]


def plain_main():
    """plaintext operations on device-resident batches, one plaintext per ciphertext vs one shared by the batch, in place, batch
    512: CKKS multiply_plain and add_plain at cfg5 and cfg2, BFV multiply_plain with a coefficient-form plaintext at cfg4 (coefficient-
    form ciphertexts: multiply_plain_normal), BGV add_plain at the cfg4 shape.  Per-ciphertext us and algorithmic GB/s: bytes that
    must cross HBM (per ciphertext: the polynomials read and written, plus its plaintext; a shared plaintext is counted once)."""
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit": os.popen(
        "nvidia-smi --query-gpu=power.limit --format=csv,noheader -i 0").read().strip()}), flush=True)
    g = torch.Generator(device="cuda")
    g.manual_seed(3)
    batch, rows = PLAIN_BATCH, []
    for cfg, scheme, n, bits, t in (("cfg5 CKKS n=65536 k=32", S.CKKS, 65536, [55] * 32, 0), ("cfg2 CKKS n=8192 k=4", S.CKKS, 8192, [54] * 4, 0),
                                    ("cfg4 BFV n=16384 k=8", S.BFV, 16384, [54] * 8, 786433),
                                    ("cfg4 shape BGV n=16384 k=8", S.BGV, 16384, [54] * 8, 786433)):
        mods = S.coeff_modulus_create(n, bits)
        L = len(mods) - 1
        ctx = S.Context(scheme, n, mods, t)
        a = rand_rows(mods, n, (batch, 2), L, g)
        word = L * n * 8
        if scheme == S.CKKS:
            plain = rand_rows(mods, n, (batch,), L, g)
            ops = [("multiply_plain", lambda cnt: ctx.d_multiply_plain_n(a, plain if cnt > 1 else plain[0], a, L, 2, batch, cnt),
                    lambda cnt: (4 * batch + (batch if cnt > 1 else 1)) * word),
                   ("add_plain", lambda cnt: ctx.d_add_plain_ntt(a, plain if cnt > 1 else plain[0], a, L, 2, batch, cnt),
                    lambda cnt: (2 * batch + (batch if cnt > 1 else 1)) * word)]
        else:
            plain = torch.randint(0, t, (batch, n), generator=g, dtype=torch.int64, device="cuda")
            if scheme == S.BFV:
                ops = [("multiply_plain (coefficient-form plaintext)",
                        lambda cnt: ctx.d_multiply_plain_coeff_n(a, plain if cnt > 1 else plain[0], a, L, 2, batch, cnt, False), None)]
            else:
                ops = [("add_plain", lambda cnt: ctx.d_add_plain_coeff_n(a, plain if cnt > 1 else plain[0], a, L, 2, batch, cnt),
                        lambda cnt: 2 * batch * word + (batch if cnt > 1 else 1) * n * 8)]
        for op, fn, nbytes in ops:
            per_ms, shared_ms = alternate([lambda: fn(batch), lambda: fn(1)])
            for form, cnt, ms in (("per-ciphertext", batch, per_ms), ("shared", 1, shared_ms)):
                res = {"config": cfg, "batch": batch, "op": op, "plaintexts": form, "us_per_ct": ms * 1e3 / batch}
                if nbytes:
                    res["GBps"] = nbytes(cnt) / (ms * 1e-3) / 1e9
                    res["of_HBM_peak"] = res["GBps"] / HBM_PEAK_GBPS
                rows.append(res)
                print(json.dumps(res), flush=True)
        del ctx, a, plain
        torch.cuda.empty_cache()
    return rows


ENCRYPT_CONFIGS = [("CKKS n=65536 k=32", S.CKKS, 65536, [55] * 32, 0, 32), ("CKKS n=8192 k=3", S.CKKS, 8192, [54] * 3, 0, 256),
                   ("BFV n=16384 k=8", S.BFV, 16384, [54] * 8, 786433, 128), ("BGV n=16384 k=8", S.BGV, 16384, [54] * 8, 786433, 128)]


def encrypt_main():
    """encryption of device-resident plaintexts at the first level, both key types: the fused entry points against the composition
    they replace (sb200_encrypt_zero_*_prng, then sb200_add_plain_ntt / sb200_add_plain_coeff_n), the same seeds, timed in
    alternating rounds; us per ciphertext and the launches of one call of each path"""
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit": os.popen(
        "nvidia-smi --query-gpu=power.limit --format=csv,noheader -i 0").read().strip()}), flush=True)
    g = torch.Generator(device="cuda")
    g.manual_seed(7)
    rows = []
    for cfg, scheme, n, bits, t, batch in ENCRYPT_CONFIGS:
        mods = S.coeff_modulus_create(n, bits)
        k, L = len(mods), len(mods) - 1
        ctx = S.Context(scheme, n, mods, t)
        rng = np.random.default_rng(11)
        sk = ctx.load_secret_key(np.stack([rng.integers(0, mods[i], n, dtype=np.uint64) for i in range(k)]))
        _, pk = ctx.generate_public_key(sk, seed=rng.integers(0, 2 ** 63, 8, dtype=np.uint64), host=False)
        seeds = rng.integers(0, 2 ** 63, (batch, 8), dtype=np.uint64)
        if scheme == S.CKKS:
            plain = rand_rows(mods, n, (batch,), L, g)
            add = lambda out: ctx.d_add_plain_ntt(out, plain, out, L, 2, batch, batch)  # noqa: E731
        else:
            plain = torch.randint(0, t, (batch, n), generator=g, dtype=torch.int64, device="cuda")
            add = lambda out: ctx.d_add_plain_coeff_n(out, plain, out, L, 2, batch, batch)  # noqa: E731
        fused_out = torch.empty((batch, 2, L, n), dtype=torch.int64, device="cuda")
        comp_out = torch.empty_like(fused_out)
        paths = {
            "symmetric": (lambda: ctx.d_encrypt_symmetric(sk, plain, fused_out, L, batch, seeds),
                          lambda: (ctx.d_encrypt_zero_symmetric(sk, comp_out, L, batch, seeds), add(comp_out))),
            "public key": (lambda: ctx.d_encrypt_asymmetric(pk, plain, fused_out, L, batch, seeds),
                           lambda: (ctx.d_encrypt_zero_asymmetric(pk, comp_out, L, batch, seeds), add(comp_out))),
        }
        for key, (fused, composed) in paths.items():
            launches = []
            for f in (fused, composed):
                c0 = ctx.launch_count
                f()
                launches.append(ctx.launch_count - c0)
            torch.cuda.synchronize()
            assert torch.equal(fused_out, comp_out), "the fused and composed paths must give the same words"
            fused_ms, comp_ms = alternate([fused, composed], rounds=3, reps=3)
            res = {"config": cfg, "batch": batch, "key": key, "fused_us_per_ct": fused_ms * 1e3 / batch,
                   "composed_us_per_ct": comp_ms * 1e3 / batch, "fused_launches": launches[0], "composed_launches": launches[1]}
            rows.append(res)
            print(json.dumps(res), flush=True)
        del ctx, sk, pk, plain, fused_out, comp_out
        torch.cuda.empty_cache()
    return rows


# the reference on ONE core (BASELINE.md section 2, survey container), ops/s, for scale only
CPU_1CORE = {
    "cfg1": {"multiply": 277.8, "relinearize": 1041.7, "multiply+relinearize": 219.3, "rotate (1 step)": 1408.5, "ct NTT+INTT": 3225.8},
    "cfg2": {"multiply": 2083.3, "relinearize": 416.7, "multiply+relinearize": 347.2, "rotate (1 step)": 434.8,
             "rescale/mod_switch": 1041.7, "ct NTT+INTT": 833.3},
    "cfg3": {"multiply": 82.6, "relinearize": 5.8, "multiply+relinearize": 5.5, "rotate (1 step)": 4.4, "rescale/mod_switch": 37.7,
             "ct NTT+INTT": 21.8},
    "cfg4": {"multiply": 19.3, "relinearize": 46.9, "multiply+relinearize": 13.7, "rotate (1 step)": 48.3, "ct NTT+INTT": 163.9},
    "cfg5": {"multiply": 21.0, "relinearize": 0.7, "multiply+relinearize": 0.7, "rotate (1 step)": 0.8, "rescale/mod_switch": 8.1,
             "ct NTT+INTT": 7.4},
}
HBM_PEAK_GBPS = 3350.0  # H100 SXM data sheet (HBM3)


def table(rows):
    """markdown table from the JSON lines main() prints"""
    out = ["# Round 1: device-resident throughput of every hot-path op at the BASELINE.json config shapes", "",
           "`python tools/bench_ops.py` on one H100 (CUDA events, 3 repetitions after a warm-up, uniform-random ciphertexts and "
           "synthetic keys resident in HBM); table written by `python tools/bench_ops.py --table <json lines>`.",
           "`cpu x1` = the reference on ONE core as measured in BASELINE.md section 2 (survey container), for scale only; "
           "the contract benchmark is bench.py.", "",
           "| config | batch | op | H100 ops/s | reference 1-core ops/s | ratio |", "|---|---|---|---|---|---|"]
    for r in rows:
        cpu = CPU_1CORE.get(r["config"][:4], {})
        for op, v in r.items():
            if op in ("config", "batch", "prng", "prng_stream_ms"):
                continue
            if "prng" in r:
                out.append(f"| {r['config']} | {r['batch']} | {r['prng']}: {op} | {v:.3g} | | |")
                continue
            if op.endswith("_GBps"):
                what = "NTT algorithmic GB/s (2*n*8 B per row per transform)" if op == "ntt_GBps" else \
                    "multiply_plain algorithmic GB/s (5*L*n*8 B per size-2 ciphertext)"
                out.append(f"| {r['config']} | {r['batch']} | {what} | {v:.0f} | | {v / HBM_PEAK_GBPS:.2f} of HBM peak |")
            else:
                c = cpu.get(op)
                out.append(f"| {r['config']} | {r['batch']} | {op} | {v:.0f} | {c if c else '-'} | {f'{v / c:.0f}x' if c else '-'} |")
    return "\n".join(out) + "\n"


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--table":
        sys.stdout.write(table([json.loads(ln) for ln in open(sys.argv[2]) if ln.startswith("{")]))
    elif len(sys.argv) == 2 and sys.argv[1] == "--prng":
        prng_main()
    elif len(sys.argv) == 2 and sys.argv[1] == "--noise-budget":
        noise_main()
    elif len(sys.argv) == 2 and sys.argv[1] == "--plain":
        plain_main()
    elif len(sys.argv) == 2 and sys.argv[1] == "--encrypt":
        encrypt_main()
    else:
        main()
