#!/usr/bin/env python3
"""Developer tool: cost of the near-best lattice (Tokenizer.lattice(margin=D) / option "lattice_margin").

    python tools/lattice_margin_bench.py [--batch 1000000] [--e2e-batch 200000] [--calls 3] [--warmup 1] [--theta 0.001]

Workload: the bench.py config-3 batch (synth-unidic dictionary, synthetic ~40-character sentences), device-resident.
Arms, each the median of --calls calls after --warmup (a host clock around a call that ends in a device
synchronisation), each with marginals off and on: lattice off, the full lattice, and the margin at D = 0 and at two D
taken from the percentiles of the positive margins of the full lattice (printed; synthetic costs have no natural
scale).  Per arm: ms per call, the "viterbi" stage (where the lattice kernels are booked), nodes per sentence and the
bytes of the node arrays.  Then end to end from pinned host memory at --e2e-batch sentences: full lattice and the
margin arms.  Checks that the tokens are the same in every arm and that each arm's flagged nodes equal them.  Prints
the GPU's name, power limit and max SM clock, read in the same run."""
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


def d2h(ptr, n, dtype):
    out = torch.empty(int(n) * np.dtype(dtype).itemsize, dtype=torch.uint8)
    if n:
        from cuda.bindings import runtime as cudart
        (err,) = cudart.cudaMemcpy(out.data_ptr(), ptr, out.numel(), cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost)
        assert int(err) == 0
    return out.numpy().view(dtype)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1000000)
    ap.add_argument("--e2e-batch", type=int, default=200000)
    ap.add_argument("--calls", type=int, default=3)
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
    print(f"batch: {n} sentences, {len(utf8) / 1e6:.1f} MB of UTF-8", flush=True)
    d_utf8 = torch.from_numpy(utf8).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()

    # D values from the positive margins of the full lattice (D = 2^62 keeps every node with a path to EOS)
    tok = vb.Tokenizer.new(d).lattice(True, margin=1 << 62)
    tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), n, len(utf8))
    nn = tok.last_device_lattice()[4]
    m = d2h(tok.last_device_lattice_margins(), nn, np.int64)
    pos = m[m > 0]
    pct = {q: int(np.percentile(pos, q)) for q in (1, 5, 25, 50)} if len(pos) else {}
    print(f"margins of the {nn} nodes with a path to EOS: {len(pos)} positive; percentiles {pct}", flush=True)
    del tok
    ds = [0] + sorted({pct.get(1, 1), pct.get(5, 1)})
    arms = [("off", False, None), ("full lattice", True, None)] + [(f"margin D={x}", True, x) for x in ds]
    for theta in (0.0, args.theta):
        for name, lat, D in arms:
            tok = vb.Tokenizer.new(d).marginals(theta).lattice(lat, margin=D)
            ms = timed(lambda: tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), n, len(utf8)),
                       args.calls, args.warmup)
            st = tok.last_stage_ms()
            line = (f"device marginals={'on ' if theta else 'off'} {name:18s} {ms:8.2f} ms/call  viterbi stage "
                    f"{st['viterbi']:7.2f} ms  launches={tok.last_launch_count()}")
            if lat:
                nn = tok.last_device_lattice()[4]
                per = 32 + (4 if theta else 0) + (8 if D is not None else 0)
                line += f"  nodes={nn} ({nn / n:.2f}/sentence)  node bytes={nn * per / 1e9:.3f} GB"
            print(line, flush=True)
            del tok

    k = min(n, args.e2e_batch)
    e_utf8 = torch.from_numpy(utf8[:int(off[k])].copy()).pin_memory().numpy()
    e_off = torch.from_numpy(off[:k + 1].astype(np.int64)).pin_memory().numpy().view(np.uint64)
    ref = None
    ok = True
    for name, lat, D in arms:
        tok = vb.Tokenizer.new(d).lattice(lat, margin=D)
        ms = timed(lambda: tok.tokenize_batch(utf8=e_utf8, byte_offsets=e_off).close(), args.calls, args.warmup)
        res = tok.tokenize_batch(utf8=e_utf8, byte_offsets=e_off)
        res.close()
        ref = res.tokens.tobytes() if ref is None else ref
        same = res.tokens.tobytes() == ref
        best = (res.nodes[(res.node_links["flags"] & vb.NODE_BEST) != 0].tobytes() == ref) if lat else True
        ok &= same and best
        extra = f"  nodes={len(res.nodes)}" if lat else ""
        print(f"e2e pinned {k} sentences {name:18s} {ms:8.2f} ms/call{extra}  tokens same: {same}  flagged = tokens: {best}",
              flush=True)
        del tok
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
