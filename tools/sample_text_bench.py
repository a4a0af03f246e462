#!/usr/bin/env python3
"""Developer tool: cost of sample text (Tokenizer.sampling(..., text=True), the option "sample_text").

    python tools/sample_text_bench.py [--batch 1000000] [--calls 5] [--warmup 1] [--theta 0.001]

Workload: the bench.py config-3 batch (synth-unidic dictionary, 1 M synthetic ~40-character sentences) from pinned
host memory, as one whole batch and through the chunked pipeline (262 144-sentence chunks).  Arms: sampling n = 1
and n = 8 without text, with -O wakati sample text and with -O mecab sample text, and best-path -O wakati for
reference.  Each time is the median of --calls calls, a host clock around a call that ends in a device
synchronisation; the "viterbi" stage (where the forward pass and the sampling kernels are booked) and the text bytes
are those of the last call.  Prints the GPU's name, power limit and max SM clock read in the same run."""
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f"nvidia-smi failed: {q.stderr.strip()}"


def timed(fn, calls, warmup):
    for _ in range(warmup):
        fn().close()
    ts = []
    for _ in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
        r.close()
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1000000)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
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
    arms = [("best wakati", 0, None)]
    for samples in (1, 8):
        arms += [(f"n={samples}", samples, None), (f"n={samples} wakati", samples, "wakati"),
                 (f"n={samples} mecab", samples, "mecab")]
    for route, chunk in (("whole", 0), ("chunked", 262144)):
        for name, samples, mode in arms:
            tok = vb.Tokenizer.new(d)
            tok.set_option("chunk_sentences", chunk)
            if samples:
                tok.sampling(samples, args.theta, 1, text=mode is not None)
            if mode or not samples:
                tok.output_mode(mode or "wakati")
            ms = timed(lambda: tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off), args.calls, args.warmup)
            st = tok.last_stage_ms()
            res = tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off)
            text_bytes = len(res.text()[1]) if (mode or not samples) else 0
            res.close()
            print(f"{route:7s} {name:12s} {ms:9.2f} ms/call  viterbi stage {st['viterbi']:7.2f} ms  "
                  f"text {text_bytes / 1e6:8.1f} MB", flush=True)
            del tok, res


if __name__ == "__main__":
    main()
