#!/usr/bin/env python3
"""Developer tool: a compact dictionary made from a MeCab model, end to end, on one GPU.

    python tools/smalldic_bench.py [--lines 1000000] [--model-lines 1000000] [--templates 16] [--runs 5]

Workload: a seeded unidic-shaped MeCab model (synth.make_mecab_model) over the connection ids of the synth-unidic
dictionary (15 626 left, 15 388 right), with --templates BIGRAM templates and --model-lines model.def lines.  The tool
times generate_bigram_info on the host (median of three calls; checked byte for byte against the Python restatement in
tests/mecab_oracle.py), builds the Matrix (synth-unidic's own matrix, bench.py config 3), Raw and Dual dictionaries, and
tokenises the bench.py config-3 corpus (--lines synthetic ~40-character sentences) with each on cuda:0: --runs timed
whole-batch calls after two warm-up calls, host clock around each call (a call returns its tokens on the host, so it
ends in a device synchronisation).  The tokens of a seeded sample of --sample sentences are compared with the oracle's
for every connector.  Prints one JSON line, with the GPU's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import vibrato_b200 as vb  # noqa: E402
from vibrato_b200 import synth  # noqa: E402
from oracle import vibrato_oracle as vo  # noqa: E402
import mecab_oracle  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    if q.returncode != 0:
        sys.exit(f"nvidia-smi failed: {q.stderr.strip()}")
    name, power, clock = (x.strip() for x in q.stdout.strip().split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=1000000)
    ap.add_argument("--model-lines", type=int, default=1000000)
    ap.add_argument("--templates", type=int, default=16)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--sample", type=int, default=2000)
    args = ap.parse_args()
    gpu = gpu_info()
    sd = synth.make_dictionary("synth-unidic")
    m = synth.make_mecab_model(sd.num_left, sd.num_right, n_templates=args.templates, n_model_lines=args.model_lines)
    src = (m["feature.def"], m["right-id.def"], m["left-id.def"], m["model.def"], 700)
    conv = []
    for _ in range(3):
        t = time.perf_counter()
        bigram = vb.generate_bigram_info(*src)
        conv.append(time.perf_counter() - t)
    oracle_bigram = mecab_oracle.generate_bigram_info(*src)
    conversion_ok = bigram == oracle_bigram
    utf8, off = synth.make_corpus(sd, args.lines, seed=20260923 + 2)  # bench.py config 3, rank 0
    rng = np.random.default_rng(20261015)
    pick = np.sort(rng.choice(args.lines, min(args.sample, args.lines), replace=False))
    b = utf8.tobytes()
    sample = [b[int(off[i]):int(off[i + 1])].decode("utf-8") for i in pick.tolist()]
    s_utf8, s_off = vb.Tokenizer.pack(sample)

    result = {"tool": "smalldic_bench", "gpu": gpu, "sentences": args.lines, "model_lines": args.model_lines,
              "templates": args.templates, "num_left": sd.num_left, "num_right": sd.num_right,
              "conversion_s": float(np.median(conv)), "conversion_matches_oracle": conversion_ok,
              "bigram_bytes": [len(x) for x in bigram], "connectors": {}}
    sample_ok = conversion_ok
    for kind in ("matrix", "raw", "dual"):
        t = time.perf_counter()
        if kind == "matrix":
            d = vb.SystemDictionaryBuilder.from_readers(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
            od = vo.OracleDictionary(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
        else:
            d = vb.SystemDictionaryBuilder.from_readers_with_bigram_info(sd.lex_csv, *bigram, sd.char_def, sd.unk_def,
                                                                         dual_connector=kind == "dual")
            od = None
        build_s = time.perf_counter() - t
        if od is None:
            od = vo.OracleDictionary(sd.lex_csv, oracle_bigram, sd.char_def, sd.unk_def, dual_connector=kind == "dual")
        tok = vb.Tokenizer.new(d, device=0)
        for _ in range(2):
            tok.tokenize_batch(utf8=utf8, byte_offsets=off)
        times = []
        for _ in range(args.runs):
            t = time.perf_counter()
            res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
            times.append(time.perf_counter() - t)
            n_tokens = res.n_tokens
            del res
        got = tok.tokenize_batch(utf8=s_utf8, byte_offsets=s_off)
        tok_off, toks = od.tokenize_batch(s_utf8, s_off, n_threads=8)[:2]
        ok = bool(np.array_equal(got.tok_offsets, tok_off) and
                  all(np.array_equal(got.tokens[n], toks[n]) for n in vb.TOKEN_DTYPE.names))
        sample_ok = sample_ok and ok
        med = float(np.median(times))
        result["connectors"][kind] = {"build_s": build_s, "call_ms_median": med * 1e3,
                                      "call_ms_min": min(times) * 1e3, "sentences_per_s": args.lines / med,
                                      "tokens": int(n_tokens), "sample_matches_oracle": ok,
                                      "viterbi": tok.describe()["last_viterbi"]}
        del tok, d, od
    result["sample_check"] = "pass" if sample_ok else "FAIL"
    print(json.dumps(result, ensure_ascii=False), flush=True)
    if not sample_ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
