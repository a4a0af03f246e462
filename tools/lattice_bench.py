#!/usr/bin/env python3
"""Developer tool: cost of lattice output (Tokenizer.lattice / option "lattice").

    python tools/lattice_bench.py [--batch 1000000] [--e2e-batch 200000] [--calls 5] [--warmup 2] [--theta 0.001]

Workload: the bench.py config-3 batch (synth-unidic dictionary, synthetic ~40-character sentences).  Arms, each the
median of --calls calls (a host clock around a call that ends in a device synchronisation):
  device-resident, --batch sentences: lattice off, lattice = 1, lattice = 1 with marginals; with the "viterbi" stage
  (where the lattice kernels are booked), the node count and the bytes of the node arrays;
  end to end from pinned host memory, --e2e-batch sentences (a size whose host result fits): lattice off and on.
Checks that the token records are the same with the lattice on and that the flagged nodes equal them.  Prints the
GPU's name and power limit read in the same run."""
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
    ap.add_argument("--e2e-batch", type=int, default=200000)
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
    print(f"batch: {n} sentences, {len(utf8) / 1e6:.1f} MB of UTF-8", flush=True)
    d_utf8 = torch.from_numpy(utf8).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    for name, lat, theta in (("off", False, 0.0), ("lattice", True, 0.0), ("lattice+marginals", True, args.theta)):
        tok = vb.Tokenizer.new(d).marginals(theta).lattice(lat)
        ms = timed(lambda: tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), n, len(utf8)), args.calls, args.warmup)
        st = tok.last_stage_ms()
        line = f"device {name:18s} {ms:8.2f} ms/call  viterbi stage {st['viterbi']:7.2f} ms  launches={tok.last_launch_count()}"
        if lat:
            nn = tok.last_device_lattice()[4]
            line += f"  nodes={nn} ({nn / n:.1f}/sentence)  node bytes={nn * (32 + (4 if theta else 0)) / 1e9:.2f} GB"
        print(line, flush=True)
        del tok

    m = min(n, args.e2e_batch)
    e_utf8 = torch.from_numpy(utf8[:int(off[m])].copy()).pin_memory().numpy()
    e_off = torch.from_numpy(off[:m + 1].astype(np.int64)).pin_memory().numpy().view(np.uint64)
    outs = {}
    for lat in (False, True):
        tok = vb.Tokenizer.new(d).lattice(lat)
        ms = timed(lambda: tok.tokenize_batch(utf8=e_utf8, byte_offsets=e_off).close(), args.calls, args.warmup)
        res = tok.tokenize_batch(utf8=e_utf8, byte_offsets=e_off)
        res.close()
        outs[lat] = res
        extra = f"  nodes={len(res.nodes)}" if lat else ""
        print(f"e2e pinned {m} sentences lattice={'on ' if lat else 'off'} {ms:8.2f} ms/call{extra}", flush=True)
        del tok
    a, b = outs[False], outs[True]
    same = a.tokens.tobytes() == b.tokens.tobytes()
    best = b.nodes[(b.node_links["flags"] & vb.NODE_BEST) != 0]
    print(f"tokens unchanged with the lattice on: {same}; flagged nodes equal the tokens: {best.tobytes() == b.tokens.tobytes()}",
          flush=True)
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
