#!/usr/bin/env python3
"""Developer tool (needs a CUDA GPU): per-call latency of small host batches, the k_small_batch route against the
default one.

    python tools/latency_bench.py [--dict synth-unidic] [--calls 2000] [--warmup 200] [--sizes 1,4,16,64,256]

Workload: the synth-unidic dictionary (vibrato_b200/synth.py; bench.py config 3) and its ~40-character synthetic
sentences.  For every batch size and both routes (the tokenizer option small_batch = the largest size, and 0) the tool
makes --calls calls of vbt_tokenize_batch through the C ABI after --warmup untimed ones, each on the next batch of a
pool of distinct batches, and takes the host clock around each call: from the call to its synchronised result in
pinned host memory, result freed.  It reports the median and p99 per size and route, the launch count and the
`last_viterbi` route of the last call (a batch over 16 KiB falls back to the default route and says so), and, as the
CPU reference point, the oracle (oracle/, one thread) per sentence.  The crossover is the smallest size at
which the default route's median is lower; the recommended "small_batch" threshold is the largest measured size below
it.  The GPU's name and power limit are read in the same run.  Prints a table and one JSON line."""
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
import vibrato_b200 as vb  # noqa: E402
from vibrato_b200 import synth  # noqa: E402
from vibrato_b200._native import check, lib  # noqa: E402
from oracle import vibrato_oracle as vo  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    if q.returncode != 0:
        sys.exit(f"nvidia-smi failed: {q.stderr.strip()}")
    name, power, clock = (x.strip() for x in q.stdout.strip().split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def stats(us):
    a = np.asarray(us)
    return {"median_us": round(float(np.median(a)), 1), "p99_us": round(float(np.percentile(a, 99)), 1)}


def time_calls(tok, pool, calls, warmup):
    """Host clock around each vbt_tokenize_batch call (it returns after the device synchronised) + result free."""
    h, L = tok.handle(), lib()
    res = C.c_void_p()
    out = []
    for i in range(warmup + calls):
        utf8, off = pool[i % len(pool)]
        t = time.perf_counter()
        check(L.vbt_tokenize_batch(h, utf8.ctypes.data, off.ctypes.data, len(off) - 1, C.byref(res)))
        L.vbt_result_free(res)
        if i >= warmup:
            out.append((time.perf_counter() - t) * 1e6)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dict", default="synth-unidic")
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--sizes", default="1,4,16,64,256")
    ap.add_argument("--oracle-calls", type=int, default=2000)
    args = ap.parse_args()
    sizes = [int(x) for x in args.sizes.split(",")]
    gpu = gpu_info()
    sd = synth.make_dictionary(args.dict)
    d = vb.SystemDictionaryBuilder.from_readers(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
    n_pool = 64  # distinct batches per size: calls cycle through them
    utf8_all, off_all = synth.make_corpus(sd, n_pool * max(sizes), seed=20260925)
    sents = [bytes(utf8_all[int(off_all[i]):int(off_all[i + 1])]) for i in range(len(off_all) - 1)]

    def pool_of(n):
        out = []
        for b in range(n_pool):
            u, o = vb.Tokenizer.pack(sents[b * n:(b + 1) * n])
            out.append((np.ascontiguousarray(u) if len(u) else np.zeros(1, np.uint8), o))
        return out

    small = vb.Tokenizer.new(d, device=0).small_batch(max(sizes))
    default = vb.Tokenizer.new(d, device=0)
    rows, result = [], {}
    for n in sizes:
        pool = pool_of(n)
        # both routes must agree on what they compute before their times mean anything
        for u, o in pool[:4]:
            a = small.tokenize_batch(utf8=u[:int(o[-1])], byte_offsets=o)
            b = default.tokenize_batch(utf8=u[:int(o[-1])], byte_offsets=o)
            if a.tokens.tobytes() != b.tokens.tobytes() or not np.array_equal(a.tok_offsets, b.tok_offsets):
                sys.exit(f"routes differ at batch size {n}")
        entry = {"bytes_mean": round(float(np.mean([int(o[-1]) for _, o in pool])), 1)}
        # alternate the two routes in rounds, so that drift in clocks or host load hits both alike
        times = {"small_batch": [], "default": []}
        per_round = max(1, args.calls // 4)
        for r in range(4):
            for name, tok in (("small_batch", small), ("default", default)):
                times[name] += time_calls(tok, pool, per_round, args.warmup if r == 0 else 20)
        for name, tok in (("small_batch", small), ("default", default)):
            entry[name] = dict(stats(times[name]), launches=tok.last_launch_count(), route=tok.describe()["last_viterbi"])
        result[str(n)] = entry
        rows.append((n, entry))
    # CPU reference point: the oracle on one thread, one sentence per call
    od = vo.OracleDictionary(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
    one = pool_of(1)
    cpu = []
    for i in range(args.oracle_calls):
        u, o = one[i % len(one)]
        t = time.perf_counter()
        od.tokenize_batch(u[:int(o[-1])], o, n_threads=1)
        cpu.append((time.perf_counter() - t) * 1e6)
    crossover = next((n for n, e in rows if e["default"]["median_us"] < e["small_batch"]["median_us"]), None)
    below = [n for n, e in rows if crossover is None or n < crossover]
    recommended = max(below) if below else 0
    print(f"{gpu['name']}, power limit {gpu['power_limit']}, max SM clock {gpu['max_sm_clock']}; dictionary {args.dict}")
    print(f"{'sentences':>9} {'bytes':>8}  {'small_batch median/p99 us (launches, route)':<48} {'default median/p99 us (launches, route)'}")
    for n, e in rows:
        s, f = e["small_batch"], e["default"]
        print(f"{n:>9} {e['bytes_mean']:>8}  {s['median_us']:>8} / {s['p99_us']:<8} ({s['launches']}, {s['route']}){'':<12}"
              f"{f['median_us']:>8} / {f['p99_us']:<8} ({f['launches']}, {f['route']})")
    print(f"oracle, one thread, per sentence: median {stats(cpu)['median_us']} us, p99 {stats(cpu)['p99_us']} us")
    print(f"crossover: {crossover}; recommended small_batch threshold: {recommended}")
    print(json.dumps({"tool": "latency_bench", "gpu": gpu, "dict": args.dict, "calls": args.calls, "sizes": result,
                      "oracle_per_sentence": stats(cpu), "crossover": crossover, "recommended_small_batch": recommended}))


if __name__ == "__main__":
    main()
