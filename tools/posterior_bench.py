#!/usr/bin/env python3
"""Developer tool: cost of posterior decoding (Tokenizer.posterior).

    python tools/posterior_bench.py [--batch 1000000] [--calls 5] [--warmup 2] [--theta 0.001] [--gamma 1]

Workload: the bench.py config-3 batch (synth-unidic dictionary, 1 M synthetic ~40-character sentences).  Arms:
marginals alone, posterior decoding at --gamma, and posterior decoding with posterior text (wakati), each
device-resident (inputs already on the GPU, results left there; the text is built on host calls only) and end to end
from pinned host memory.  Each time is the median of --calls calls, a host clock around a call that ends in a device
synchronisation; the "viterbi" stage (where the posterior kernels are booked) is last_stage_ms() of the last call.
Also prints tokens per sentence of the best and the posterior paths and the share of sentences whose posterior path
differs from the best path, checks that tokens and marginals are byte-identical across the arms, and prints the GPU's
name, power limit and max SM clock read in the same run."""
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
    ap.add_argument("--gamma", type=float, default=1.0)
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

    ref = None
    for arm in ("marginals alone", "posterior", "posterior text"):
        tok = vb.Tokenizer.new(d).marginals(args.theta)
        if arm != "marginals alone":
            tok.posterior(args.gamma, text=arm == "posterior text")
        if arm == "posterior text":
            tok.output_mode("wakati")
        res = tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off)
        res.close()
        outs = (res.tokens.tobytes(), res.token_probs.tobytes(), res.path_probs.tobytes())
        if ref is None:
            ref = outs
        elif outs != ref:
            sys.exit(f"{arm}: tokens or marginals differ from marginals alone")
        if arm == "posterior":
            toff, poff = res.tok_offsets.astype(np.int64), res.posterior_offsets.astype(np.int64)
            cols = ["start_char", "end_char", "word_idx"]
            best = res.tokens[cols]
            post = res.posterior_tokens[cols]
            differ = sum(1 for i in range(n) if toff[i + 1] - toff[i] != poff[i + 1] - poff[i] or
                         best[toff[i]:toff[i + 1]].tobytes() != post[poff[i]:poff[i + 1]].tobytes())
            print(f"tokens per sentence: best path {toff[-1] / n:.3f}, posterior path {poff[-1] / n:.3f}; "
                  f"posterior path differs from the best path in {differ} of {n} sentences ({100.0 * differ / n:.2f}%)",
                  flush=True)
        del res
        arms = [("device", lambda: tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), n, len(utf8))),
                ("e2e", lambda: tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off))]
        if arm == "posterior text":
            arms = arms[1:]  # device-resident calls build no text
        for route, fn in arms:
            ms = timed(fn, args.calls, args.warmup)
            st = tok.last_stage_ms()
            print(f"{arm:16s} {route:6s} {ms:8.2f} ms/call  viterbi stage {st['viterbi']:7.2f} ms  "
                  f"launches={tok.last_launch_count()}", flush=True)
        del tok, arms, fn  # one tokenizer's workspace at a time
    print("tokens and marginals byte-identical across the arms: True", flush=True)


if __name__ == "__main__":
    main()
