#!/usr/bin/env python3
"""Developer tool: end-to-end time of the output formats (Tokenizer.output_format) against the fixed output modes.

    python tools/format_bench.py [--batch 1000000] [--calls 5] [--warmup 2]

Workload: the bench.py config-3 batch (synth-unidic dictionary, 1 M synthetic ~40-character sentences), from pinned
host memory, on the whole-batch route (chunk_sentences = 0) and the chunked pipeline (its default).  Arms:
    mode mecab   vs  '%m\\t%H\\n'      (the same bytes: checked)
    mode wakati  vs  '%m '
    '%f[6] '                           (lemmatised wakati: one field per token)
    '%m\\t%f[0,1]\\t%pc\\t%pC\\n'         (fields and costs)
Each time is the median of --calls calls, a host clock around a call that ends with the text on the host.  Prints
text bytes, ms per call, the field-table size and build time of each format, and the GPU's name and power limit read
in the same run."""
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

ARMS = [("mode", "mecab"), ("format", "%m\\t%H\\n"), ("mode", "wakati"), ("format", "%m "), ("format", "%f[6] "),
        ("format", "%m\\t%f[0,1]\\t%pc\\t%pC\\n")]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f"nvidia-smi failed: {q.stderr.strip()}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1000000)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if torch.cuda.device_count() == 0:
        sys.exit("no CUDA device: this tool measures GPU time")
    print("gpu:", gpu_info().replace("\n", " | "), flush=True)
    sd = synth.make_dictionary("synth-unidic")
    utf8, off = synth.make_corpus(sd, args.batch, seed=20260923 + 2)  # bench.py config 3, rank 0
    d = vb.SystemDictionaryBuilder.from_readers(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
    h_utf8 = torch.from_numpy(utf8).pin_memory().numpy()
    h_off = torch.from_numpy(off.astype(np.int64)).pin_memory().numpy().view(np.uint64)
    print(f"batch: {args.batch} sentences, {len(utf8) / 1e6:.1f} MB of UTF-8", flush=True)
    for route, chunk in (("whole", 0), ("chunked", None)):
        tok = vb.Tokenizer.new(d)
        if chunk is not None:
            tok.set_option("chunk_sentences", chunk)
        mecab = None
        for kind, arg in ARMS:
            if kind == "mode":
                tok.output_mode(arg)
                table = ""
            else:
                tok.output_format(arg)
                ft = tok.describe().get("field_table", {})
                table = f"  field_table={ft.get('bytes', 0) / 1e6:.1f} MB built in {ft.get('build_ms', 0.0):.2f} ms"
            for _ in range(args.warmup):
                tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off).close()
            times = []
            for _ in range(args.calls):
                t = time.perf_counter()
                r = tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off)
                times.append(time.perf_counter() - t)
                if len(times) < args.calls:
                    r.close()
            toff, text = r.text()
            r.close()
            if arg == "mecab":
                mecab = (toff, text)
            same = ""
            if arg == "%m\\t%H\\n":
                same = f"  identical_to_mecab={np.array_equal(toff, mecab[0]) and text == mecab[1]}"
            ms = np.array(times) * 1e3
            print(f"route={route:7s} {kind:6s} {arg!r:30s} ms/call median={np.median(ms):8.2f} min={ms.min():8.2f} "
                  f"max={ms.max():8.2f}  text={len(text) / 1e6:8.1f} MB{table}{same}", flush=True)
        del tok
    print("gpu:", gpu_info().replace("\n", " | "), flush=True)


if __name__ == "__main__":
    main()
