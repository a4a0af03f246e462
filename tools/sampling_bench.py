#!/usr/bin/env python3
"""Developer tool: cost of segmentation sampling (Tokenizer.sampling / vbt_tokenizer_set_sampling).

    python tools/sampling_bench.py [--batch 1000000] [--calls 5] [--warmup 2] [--theta 0.001]

Workload: the bench.py config-3 batch (synth-unidic dictionary, 1 M synthetic ~40-character sentences).  Arms:
sampling off, n = 1 and n = 8, and marginals on (for comparison), each device-resident (inputs already on the GPU,
results left there) and end to end from pinned host memory as one whole batch.  Each time is the median of --calls
calls, a host clock around a call that ends in a device synchronisation; the "viterbi" stage (where the forward pass
and the sampling kernels are booked) is last_stage_ms() of the last call.  Prints the sample tokens and bytes, checks
that the token records with sampling on equal those with it off, and prints the GPU's name and power limit read in
the same run."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import vibrato_b200 as vb  # noqa: E402
from vibrato_b200 import synth  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f"nvidia-smi failed: {q.stderr.strip()}"


def timed(fn, calls, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1000000)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--theta", type=float, default=0.001)
    args = ap.parse_args()
    if torch.cuda.device_count() == 0:
        sys.exit("no CUDA device: this tool measures GPU time")
    print("gpu:", gpu_info().replace("\n", " | "), flush=True)
    sd = synth.make_dictionary("synth-unidic")
    utf8, off = synth.make_corpus(sd, args.batch, seed=20260923 + 2)  # bench.py config 3, rank 0
    d = vb.SystemDictionaryBuilder.from_readers(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
    n = len(off) - 1
    print(f"batch: {n} sentences, {len(utf8) / 1e6:.1f} MB of UTF-8, theta {args.theta}", flush=True)
    h_utf8 = torch.from_numpy(utf8).pin_memory().numpy()
    h_off = torch.from_numpy(off.astype(np.int64)).pin_memory().numpy().view(np.uint64)
    d_utf8 = torch.from_numpy(utf8).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()

    tokens = {}
    for name, samples, marg in (("off", 0, False), ("n=1", 1, False), ("n=8", 8, False), ("marginals", 0, True)):
        tok = vb.Tokenizer.new(d)
        tok.set_option("chunk_sentences", 0)
        if samples:
            tok.sampling(samples, args.theta, 1)
        if marg:
            tok.marginals(args.theta)
        res = tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off)
        res.close()
        tokens[name] = (res.tok_offsets, res.tokens)
        extra = ""
        if samples:
            nst = len(res.samples)
            extra = f"  sample tokens {nst} ({nst / n / samples:.2f} per sample), {nst * 24 / 1e9:.2f} GB"
        del res
        for route, fn in (("device", lambda: tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), n, len(utf8))),
                          ("e2e", lambda: tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off))):
            ms = timed(fn, args.calls, args.warmup)
            st = tok.last_stage_ms()
            print(f"{name:9s} {route:6s} {ms:8.2f} ms/call  viterbi stage {st['viterbi']:7.2f} ms  "
                  f"launches={tok.last_launch_count()}{extra if route == 'device' else ''}", flush=True)
        del tok, fn
    for name in ("n=1", "n=8", "marginals"):
        same = np.array_equal(tokens[name][0], tokens["off"][0]) and tokens[name][1].tobytes() == tokens["off"][1].tobytes()
        print(f"token records with {name}: {'equal to' if same else 'DIFFERENT FROM'} sampling off", flush=True)
        if not same:
            sys.exit(1)


if __name__ == "__main__":
    main()
