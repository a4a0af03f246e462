#!/usr/bin/env python3
"""Developer tool: cost of marginal probabilities (Tokenizer.marginals / vbt_tokenizer_set_marginals).

    python tools/marginal_bench.py [--batch 1000000] [--calls 5] [--warmup 2] [--theta 0.001] [--oracle-sample 2000]

Workload: the bench.py config-3 batch (synth-unidic dictionary, 1 M synthetic ~40-character sentences).  Arms:
marginals off and on, each device-resident (inputs already on the GPU, results left there) and end to end from
pinned host memory, as one whole batch and through the chunked host pipeline.  Each time is the median of --calls
calls, a host clock around a call that ends in a device synchronisation; the "viterbi" stage (where the two marginal
kernels are booked) is last_stage_ms() of the last call.  The token records with marginals on must equal those with
them off; the probabilities of a seeded sample of --oracle-sample sentences are compared with the forward-backward
restatement (tests/marginal_oracle.py) and the largest relative error is printed.  Prints the GPU's name and power
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
    ap.add_argument("--oracle-sample", type=int, default=2000)
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

    results = {}
    for chunk in (0, 262144):
        for theta in (0.0, args.theta):
            tok = vb.Tokenizer.new(d)
            tok.set_option("chunk_sentences", chunk)
            tok.marginals(theta)
            res = tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off)
            res.close()  # keeps copies of the arrays, frees the pinned result
            results[(chunk, theta)] = (res.tok_offsets, res.tokens, res.token_probs, res.path_probs)
            del res
            arms = [("e2e", lambda: tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off))]
            if chunk == 0:
                arms.append(("device", lambda: tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), n, len(utf8))))
            for route, fn in arms:
                ms = timed(fn, args.calls, args.warmup)
                st = tok.last_stage_ms()
                print(f"{'whole' if chunk == 0 else 'chunked':7s} {route:6s} marginals={'on ' if theta else 'off'} "
                      f"{ms:8.2f} ms/call  viterbi stage {st['viterbi']:7.2f} ms  launches={tok.last_launch_count()}",
                      flush=True)
            del tok, arms, fn  # one tokenizer's workspace at a time
    for chunk in (0, 262144):
        a, b = results[(chunk, 0.0)], results[(chunk, args.theta)]
        same = np.array_equal(a[0], b[0]) and a[1].tobytes() == b[1].tobytes()
        print(f"{'whole' if chunk == 0 else 'chunked'}: token records with marginals on "
              f"{'equal' if same else 'DIFFER FROM'} those with them off ({len(a[1])} tokens)", flush=True)
        if not same:
            sys.exit(1)
    w, c = results[(0, args.theta)], results[(262144, args.theta)]
    print("whole vs chunked probabilities bit-identical:",
          w[2].tobytes() == c[2].tobytes() and w[3].tobytes() == c[3].tobytes(),
          flush=True)

    if args.oracle_sample:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import marginal_oracle as mo
        from bounded_oracle import BoundedOracle
        from oracle import vibrato_oracle as vo
        od = vo.OracleDictionary(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
        bo = BoundedOracle(od, sd.char_def, sd.unk_def)
        rng = np.random.default_rng(7)
        worst = 0.0
        for i in sorted(rng.choice(n, size=min(n, args.oracle_sample), replace=False).tolist()):
            s = utf8[off[i]:off[i + 1]].tobytes()
            tp, pp = mo.sentence_marginals(bo, s, args.theta)
            a, b = int(w[0][i]), int(w[0][i + 1])
            got = np.concatenate([w[2][a:b], [w[3][i]]]).astype(np.float64)
            exp = np.array(tp + [pp], dtype=np.float64)
            worst = max(worst, float(np.max(np.abs(got - exp) / np.maximum(exp, 1e-6))))
        print(f"oracle sample: {args.oracle_sample} sentences, max |GPU - restatement| / max(p, 1e-6) = {worst:.3e}", flush=True)


if __name__ == "__main__":
    main()
