#!/usr/bin/env python3
"""Developer tool: cost of required tokens (vbt_tokenize_batch_spans / _device_spans).

    python tools/span_bench.py [--batch 1000000] [--calls 5] [--warmup 2]

Workload: the bench.py config-3 batch (synth-unidic dictionary, 1 M synthetic ~40-character sentences).  Arms:
    no_spans      the plain call
    empty         every span list empty (runs the plain kernels; must give the plain tokens)
    one           one span per sentence over its middle best-path token, without a pattern
    one_pattern   the same span with a two-field pattern (the token's first two feature fields)
    forced        every best-path token of every sentence as a span (forced alignment)
each device-resident (inputs and span lists already on the GPU, results left there) and end to end (pinned host
memory in, tokens on the host).  "empty" must give the plain tokens.  The other arms keep the best path in the
constrained lattice, but a span's ends are boundaries, which may admit unknown words a crossing lexicon word used to
suppress; the tool reports sentences whose token ranges differ from the plain call.  Each time is the median of --calls calls, a
host clock around a call that ends in a device synchronisation; the stage times are last_stage_ms() of the last call.
Prints the GPU's name and power limit read in the same run."""
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


def pinned(a):
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()


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
    dic = vb.SystemDictionaryBuilder.from_readers(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
    n = len(off) - 1
    print(f"batch: {n} sentences, {len(utf8) / 1e6:.1f} MB of UTF-8", flush=True)
    tok = vb.Tokenizer.new(dic)
    h_utf8, h_off = pinned(utf8), pinned(off.astype(np.uint64))
    d_utf8 = torch.from_numpy(utf8).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    base = tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off)
    t_off, toks = base.tok_offsets.astype(np.int64), base.tokens.copy()
    counts = np.diff(t_off)
    has = counts > 0
    mid = t_off[:-1] + counts // 2  # the middle token of each sentence (unused where a sentence has none)
    one_off = np.zeros(n + 1, dtype=np.uint64)
    one_off[1:] = np.cumsum(has)
    sel = mid[has]
    one = np.stack([toks["start_byte"][sel], toks["end_byte"][sel], np.full(len(sel), vb.SPAN_ANY, np.uint32)], 1)
    words, inv = np.unique(toks["word_idx"][sel], return_inverse=True)
    pats = [",".join(dic.word_feature(int(w)).split(",")[:2]) for w in words]
    one_pat = one.copy()
    one_pat[:, 2] = inv.astype(np.uint32)
    forced = np.stack([toks["start_byte"], toks["end_byte"], np.full(len(toks), vb.SPAN_ANY, np.uint32)], 1)
    arms = {
        "no_spans": None,
        "empty": (np.zeros(n + 1, dtype=np.uint64), np.zeros((0, 3), np.uint32), []),
        "one": (one_off, one.astype(np.uint32), []),
        "one_pattern": (one_off, one_pat.astype(np.uint32), pats),
        "forced": (t_off.astype(np.uint64), forced.astype(np.uint32), []),
    }
    for name, lists in arms.items():
        if lists is None:
            e2e = lambda: tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off)  # noqa: E731
            dev = lambda: tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), n, len(utf8))  # noqa: E731
            n_spans = 0
        else:
            so, recs, pt = pinned(lists[0]), pinned(lists[1]), lists[2]
            d_so = torch.from_numpy(lists[0].view(np.int64)).cuda()
            d_sp = (torch.from_numpy(lists[1].reshape(-1).view(np.int32)).cuda() if len(lists[1])
                    else torch.zeros(3, dtype=torch.int32, device="cuda"))
            n_spans = len(lists[1])
            e2e = lambda so=so, recs=recs, pt=pt: tok.tokenize_batch(  # noqa: E731
                utf8=h_utf8, byte_offsets=h_off, span_offsets=so, span_records=recs, patterns=pt)
            dev = lambda d_so=d_so, d_sp=d_sp, ns=n_spans, pt=pt: tok.tokenize_batch_device(  # noqa: E731
                d_utf8.data_ptr(), d_off.data_ptr(), n, len(utf8), d_span_offsets=d_so.data_ptr(),
                d_spans=d_sp.data_ptr(), n_spans=ns, patterns=pt)
            r = e2e()
            if name == "empty" and r.tokens.tobytes() != toks.tobytes():
                sys.exit("empty: the tokens differ from the plain call")
            if not np.array_equal(r.tok_offsets, base.tok_offsets):
                print(f"{name}: token counts differ in {int(np.sum(np.diff(r.tok_offsets.astype(np.int64)) != counts))} "
                      "sentences", flush=True)
            elif not (np.array_equal(r.tokens["start_byte"], toks["start_byte"]) and
                      np.array_equal(r.tokens["end_byte"], toks["end_byte"])):
                print(f"{name}: same token counts, some ranges differ", flush=True)
        for route, fn in (("device", dev), ("e2e", e2e)):
            ms = timed(fn, args.calls, args.warmup)
            st = {k: round(v, 3) for k, v in tok.last_stage_ms().items()}
            print(f"{name:12s} {route:6s} spans={n_spans:>9d} {ms:8.2f} ms/call  viterbi={st['viterbi']}  "
                  f"candidates={st['candidates']}  decode={st['decode']}  launches={tok.last_launch_count()}", flush=True)


if __name__ == "__main__":
    main()
