#!/usr/bin/env python3
"""Developer tool: end-to-end time of the output stage (Tokenizer.output_mode) on each host route.

    python tools/output_bench.py [--batch 1000000] [--calls 5] [--warmup 2] [--modes wakati,mecab]

Workload: the bench.py config-3 batch (synth-unidic dictionary, 1 M synthetic ~40-character sentences), from pinned
host memory.  Arms, per mode:
    whole    single device, chunk_sentences = 0 (the batch runs as one piece, one synchronisation to size the text)
    chunked  single device, chunk_sentences at its default (the three-stream pipeline)
    devN     one tokenizer over devices 0..N-1, for every N up to the GPUs present
Each arm's time is a host clock around a call that ends in the result being on the host (the call synchronises).
Prints ms per call and text bytes per second, checks that every arm's text is byte-identical to the whole-batch
arm's, and prints the GPU's name and power limit read in the same run."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1000000)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--modes", default="wakati,mecab")
    args = ap.parse_args()
    n_gpu = torch.cuda.device_count()
    if n_gpu == 0:
        sys.exit("no CUDA device: this tool measures GPU time")
    print("gpus:", gpu_info().replace("\n", " | "), flush=True)
    sd = synth.make_dictionary("synth-unidic")
    utf8, off = synth.make_corpus(sd, args.batch, seed=20260923 + 2)  # bench.py config 3, rank 0
    d = vb.SystemDictionaryBuilder.from_readers(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
    h_utf8 = torch.from_numpy(utf8).pin_memory().numpy()
    h_off = torch.from_numpy(off.astype(np.int64)).pin_memory().numpy().view(np.uint64)
    print(f"batch: {args.batch} sentences, {len(utf8) / 1e6:.1f} MB of UTF-8", flush=True)

    def arms():
        whole = vb.Tokenizer.new(d)
        whole.set_option("chunk_sentences", 0)
        yield "whole", whole
        yield "chunked", vb.Tokenizer.new(d)
        for n in range(1, n_gpu + 1):
            yield f"dev{n}", vb.Tokenizer.new(d, devices=list(range(n)))

    for mode in args.modes.split(","):
        ref = None
        for name, tok in arms():
            tok.output_mode(mode)
            for _ in range(args.warmup):
                tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off).close()
            times = []
            for _ in range(args.calls):
                t = time.perf_counter()
                r = tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off)
                times.append(time.perf_counter() - t)
                r.close()
            r = tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off)
            toff, text = r.text()
            r.close()
            if ref is None:
                ref = (toff, text)
            same = np.array_equal(toff, ref[0]) and text == ref[1]
            ms = np.array(times) * 1e3
            print(f"mode={mode:6s} arm={name:8s} ms/call median={np.median(ms):8.2f} min={ms.min():8.2f} "
                  f"max={ms.max():8.2f}  text={len(text) / 1e6:8.1f} MB  {len(text) / 1e9 / (np.median(ms) * 1e-3):6.2f} GB/s"
                  f"  identical_to_whole={same}", flush=True)
            if not same:
                sys.exit(f"{name} text differs from the whole-batch text ({mode})")
            del tok
    print("gpus:", gpu_info().replace("\n", " | "), flush=True)


if __name__ == "__main__":
    main()
