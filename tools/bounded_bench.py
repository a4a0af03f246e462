#!/usr/bin/env python3
"""Developer tool: cost of required boundaries (vbt_tokenize_batch_bounded / _device_bounded).

    python tools/bounded_bench.py [--batch 1000000] [--calls 5] [--warmup 2]

Workload: the bench.py config-3 batch (synth-unidic dictionary, 1 M synthetic ~40-character sentences).  Arms:
    unbounded            the plain call
    (a) empty            every boundary list empty (runs the unbounded kernels)
    (b) own              each sentence's boundaries = the end bytes of its unbounded tokens
    (c) every4           a boundary every 4 characters
each device-resident (inputs and boundary lists already on the GPU, results left there) and end to end (pinned host
memory in, tokens on the host).  Each time is the median of --calls calls, a host clock around a call that ends in a
device synchronisation; the stage times are last_stage_ms() of the last call.  (a) must give the unbounded tokens.
(b) keeps the unbounded path in the constrained lattice but may also add candidates (a lexicon word that crossed a
boundary no longer suppresses unknown words), so its tokens can differ: the tool counts the sentences that differ and
checks --oracle-sample of them against the bounded oracle (tests/bounded_oracle.py).  Prints the GPU's name and power
limit read in the same run."""
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


def every_k_chars(d_utf8, d_off, k):
    """Boundary CSR (device tensors) with a boundary in front of every k-th character of each sentence."""
    n_bytes = d_utf8.numel()
    pos = torch.arange(n_bytes, device="cuda", dtype=torch.int64)
    lead = (d_utf8 & 0xC0) != 0x80
    cum = torch.cumsum(lead.to(torch.int64), 0)  # characters up to and including each byte
    sent = torch.searchsorted(d_off[1:], pos, right=True)
    first = d_off[:-1]
    cbase = torch.where(first > 0, cum[(first - 1).clamp(min=0)], torch.zeros_like(first))
    local = cum - 1 - cbase[sent]  # character index of a lead byte inside its sentence
    sel = lead & (local % k == 0) & (local > 0)
    bnd = (pos - d_off[sent])[sel].to(torch.int32)
    counts = torch.bincount(sent[sel], minlength=d_off.numel() - 1)
    b_off = torch.zeros(d_off.numel(), dtype=torch.int64, device="cuda")
    b_off[1:] = torch.cumsum(counts, 0)
    return b_off, bnd


def oracle_for(sd):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from bounded_oracle import BoundedOracle
    from oracle import vibrato_oracle as vo
    od = vo.OracleDictionary(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
    return BoundedOracle(od, sd.char_def, sd.unk_def)


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
    ap.add_argument("--oracle-sample", type=int, default=200)
    args = ap.parse_args()
    if torch.cuda.device_count() == 0:
        sys.exit("no CUDA device: this tool measures GPU time")
    print("gpu:", gpu_info().replace("\n", " | "), flush=True)
    sd = synth.make_dictionary("synth-unidic")
    utf8, off = synth.make_corpus(sd, args.batch, seed=20260923 + 2)  # bench.py config 3, rank 0
    d = vb.SystemDictionaryBuilder.from_readers(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
    n = len(off) - 1
    print(f"batch: {n} sentences, {len(utf8) / 1e6:.1f} MB of UTF-8", flush=True)
    tok = vb.Tokenizer.new(d)
    h_utf8 = torch.from_numpy(utf8).pin_memory().numpy()
    h_off = torch.from_numpy(off.astype(np.int64)).pin_memory().numpy().view(np.uint64)
    d_utf8 = torch.from_numpy(utf8).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()

    base = tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off)
    b_tok_off, b_toks = base.tok_offsets.copy(), base.tokens.copy()
    empty_off = np.zeros(n + 1, dtype=np.uint64)
    arms = {
        "unbounded": None,
        "a_empty": (empty_off, np.zeros(0, dtype=np.uint32)),
        "b_own": (b_tok_off.astype(np.uint64), b_toks["end_byte"].astype(np.uint32)),
    }
    c_off, c_bnd = every_k_chars(d_utf8, d_off, 4)
    arms["c_every4"] = (c_off.cpu().numpy().astype(np.uint64), c_bnd.cpu().numpy().astype(np.uint32))
    for name, lists in arms.items():
        if lists is None:
            e2e = lambda: tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off)  # noqa: E731
            dev = lambda: tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), n, len(utf8))  # noqa: E731
            n_bnd = 0
        else:
            bo = torch.from_numpy(lists[0].view(np.int64)).pin_memory().numpy().view(np.uint64)
            bv = torch.from_numpy(lists[1].view(np.int32)).pin_memory().numpy().view(np.uint32)
            d_bo = torch.from_numpy(lists[0].view(np.int64)).cuda()
            d_bv = torch.from_numpy(lists[1].view(np.int32)).cuda() if len(lists[1]) else torch.zeros(1, dtype=torch.int32,
                                                                                                      device="cuda")
            n_bnd = len(lists[1])
            e2e = lambda bo=bo, bv=bv: tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off, bnd_offsets=bo, bnd=bv)  # noqa: E731
            dev = lambda d_bo=d_bo, d_bv=d_bv, nb=n_bnd: tok.tokenize_batch_device(  # noqa: E731
                d_utf8.data_ptr(), d_off.data_ptr(), n, len(utf8), d_bnd_offsets=d_bo.data_ptr(), d_bnd=d_bv.data_ptr(),
                n_bnd=nb)
        if name == "a_empty":
            r = e2e()
            if not (np.array_equal(r.tok_offsets, b_tok_off) and r.tokens.tobytes() == b_toks.tobytes()):
                sys.exit("empty lists changed the tokens")
            print("a_empty: tokens equal to the unbounded call", flush=True)
        if name == "b_own":
            r = e2e()
            differ = [i for i in range(n) if not np.array_equal(
                r.tokens[r.tok_offsets[i]:r.tok_offsets[i + 1]].tobytes(), b_toks[b_tok_off[i]:b_tok_off[i + 1]].tobytes())]
            sample = (differ + list(range(n)))[:args.oracle_sample]
            oracle = oracle_for(sd)
            for i in sample:
                s = utf8[off[i]:off[i + 1]].tobytes()
                own = b_toks["end_byte"][b_tok_off[i]:b_tok_off[i + 1]].tolist()
                if oracle.tokenize(s, own).tobytes() != r.tokens[r.tok_offsets[i]:r.tok_offsets[i + 1]].tobytes():
                    sys.exit(f"b_own: sentence {i} differs from the bounded oracle")
            print(f"b_own: {len(differ)} of {n} sentences differ from the unbounded tokens; {len(sample)} checked "
                  f"against the bounded oracle (the differing ones first): equal", flush=True)
        for route, fn in (("device", dev), ("e2e", e2e)):
            ms = timed(fn, args.calls, args.warmup)
            st = {k: round(v, 3) for k, v in tok.last_stage_ms().items()}
            print(f"{name:10s} {route:6s} boundaries={n_bnd:>9d} {ms:8.2f} ms/call  launches={tok.last_launch_count()}"
                  f"  stages={st}", flush=True)


if __name__ == "__main__":
    main()
