#!/usr/bin/env python3
"""Developer tool: wall time of the `reorder` and `tokenize -O wakati` CLIs on the bench.py config-3 corpus.

    python tools/dict_tools_bench.py [--lines 1000000] [--runs 2] [--level 3]

Workload: the synth-unidic dictionary, written once as `system.dic.zst` (Dictionary.write_zstd_file at --level; the
level changes the file size, not what the tools read), and the config-3 corpus (1 M synthetic ~40-character
sentences, one per line) as a file on stdin.  Each tool's time is a host clock around the whole process: dictionary
load and upload, tokenisation, and its output (`tokenize` writes to /dev/null, `reorder` its two mapping files).  The
same tool on an empty stdin gives the fixed part (load + upload).  Prints the GPU's name and power limit read in the
same run.  Everything is written to a temporary directory."""
import argparse
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import vibrato_b200 as vb  # noqa: E402
from vibrato_b200 import synth  # noqa: E402

BIN = os.path.join(ROOT, "vibrato_b200", "bin")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f"nvidia-smi failed: {q.stderr.strip()}"


def timed(argv, stdin_path):
    with open(stdin_path, "rb") as fin:
        t = time.perf_counter()
        p = subprocess.run(argv, stdin=fin, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
        dt = time.perf_counter() - t
    if p.returncode != 0:
        sys.exit(f"{argv[0]} failed: {p.stderr.decode(errors='replace')}")
    return dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=1000000)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--level", type=int, default=3)
    args = ap.parse_args()
    print("gpus:", gpu_info().replace("\n", " | "), flush=True)
    sd = synth.make_dictionary("synth-unidic")
    utf8, off = synth.make_corpus(sd, args.lines, seed=20260923 + 2)  # bench.py config 3, rank 0
    with tempfile.TemporaryDirectory() as tmp:
        corpus, empty, dic = os.path.join(tmp, "corpus.txt"), os.path.join(tmp, "empty.txt"), os.path.join(tmp, "system.dic.zst")
        b = utf8.tobytes()
        with open(corpus, "wb") as f:
            f.write(b"".join(b[int(off[i]):int(off[i + 1])] + b"\n" for i in range(args.lines)))
        open(empty, "wb").close()
        d = vb.SystemDictionaryBuilder.from_readers(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
        t = time.perf_counter()
        d.write_zstd_file(dic, args.level)
        print(f"write_zstd_file level {args.level}: {time.perf_counter() - t:.2f} s, {os.path.getsize(dic) / 1e6:.1f} MB "
              f"(stream {len(d.write()) / 1e6:.1f} MB); corpus {os.path.getsize(corpus) / 1e6:.1f} MB, {args.lines} lines",
              flush=True)
        del d
        tools = {"reorder": [os.path.join(BIN, "reorder"), "-i", dic, "-o", os.path.join(tmp, "reordered")],
                 "tokenize -O wakati": [os.path.join(BIN, "tokenize"), "-i", dic, "-O", "wakati"]}
        for name, argv in tools.items():
            for _ in range(args.runs):
                full, fixed = timed(argv, corpus), timed(argv, empty)
                print(f"{name:20s} wall {full:7.2f} s  (empty stdin {fixed:6.2f} s; the {args.lines} lines add "
                      f"{full - fixed:6.2f} s)", flush=True)
    print("gpus:", gpu_info().replace("\n", " | "), flush=True)


if __name__ == "__main__":
    main()
