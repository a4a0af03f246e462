#!/usr/bin/env python3
"""Bytes of the candidate pool per batch, as 16-byte candidate records and as 8-byte segments (CPU only).

    python tools/pool_bytes.py [--config 3] [--sample 2000]

K2 (k_candidates) stores, for every start position, the sources of its candidates: one segment per trie hit (a
postings list) and one per unknown-word span (the unk.def entries of a category).  This tool rebuilds those sources
for a seeded sample of a bench.py corpus with the oracle (oracle/, common-prefix search and CharInfo) and
Tokenizer::add_lattice_edges' unknown-word rules, counts candidates and segments per position, and scales them to
the configuration's batch.  Counts only: no timing.  Prints a short table and one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vibrato_b200 import synth  # noqa: E402
from oracle import vibrato_oracle as vo  # noqa: E402
import bench  # noqa: E402  (CONFIGS only)


def _text(x):
    return x.decode() if isinstance(x, (bytes, bytearray)) else x


def unk_entries_per_category(char_def, unk_def):
    """unk.def entries per category id (the order of the category lines of char.def)."""
    names = []
    for line in _text(char_def).splitlines():
        t = line.split("#")[0].split()
        if t and not t[0].startswith("0x"):
            names.append(t[0])
    per = {n: 0 for n in names}
    for line in _text(unk_def).splitlines():
        if line.strip():
            per[line.split(",")[0]] = per.get(line.split(",")[0], 0) + 1
    return [per[n] for n in names]


def position_sources(od, text, p, groupable, ne_of, max_grouping=None):
    """(candidates, segments) of start position p: user lexicon absent, system trie hits, then unknown spans."""
    hits = od.common_prefix(text[p:], 0)
    n_words = len(hits)
    n_hits = len({end for _, end in hits})
    ci = od.char_info(ord(text[p]))
    invoke, group, length, base = (ci >> 26) & 1, (ci >> 27) & 1, ci >> 28, (ci >> 18) & 0xFF
    ne = ne_of[base]
    spans = 0
    matched = n_words != 0
    if not (matched and not invoke):  # unknown.rs:69-116
        g = groupable[p]
        if group and (max_grouping is None or g - 1 <= max_grouping):
            spans += 1
            matched = True
        for i in range(1, min(length, g) + 1):
            if group and i == g:
                continue
            spans += 1
            matched = True
        if not matched:
            spans += 1
    if ne == 0:
        spans = 0
    return n_words + spans * ne, n_hits + spans


def groupable_of(od, text):
    cats = [od.char_info(ord(c)) & 0x3FFFF for c in text]
    n = len(text)
    g = [0] * n
    run_end = n
    for c in range(n - 1, -1, -1):
        if c + 1 == n or (cats[c] & cats[c + 1]) == 0:
            run_end = c + 1
        g[c] = run_end - c
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=3, choices=sorted(bench.CONFIGS))
    ap.add_argument("--sample", type=int, default=2000)
    args = ap.parse_args()
    cfg = bench.CONFIGS[args.config]
    sd = synth.make_dictionary(cfg["dict"], with_matrix=True)
    od = vo.OracleDictionary(sd.lex_csv, sd.matrix_def(), sd.char_def, sd.unk_def)
    ne_of = unk_entries_per_category(sd.char_def, sd.unk_def)
    kw = dict(cfg["corpus"])
    if cfg["user"]:
        sys.exit("configurations with a user lexicon are not covered")
    utf8, off = synth.make_corpus(sd, args.sample, seed=20260923 + 2, **kw)
    cands = segs = positions = 0
    seg_hist = {}
    for s in range(args.sample):
        text = bytes(utf8[off[s]:off[s + 1]]).decode()
        g = groupable_of(od, text)
        for p in range(len(text)):
            c, k = position_sources(od, text, p, g, ne_of)
            cands += c
            segs += k
            positions += 1
            seg_hist[k] = seg_hist.get(k, 0) + 1
    scale = cfg["batch"] / args.sample
    old_b, new_b = cands * 16 * scale, segs * 8 * scale
    res = {
        "config": args.config, "sample": args.sample, "positions": positions,
        "candidates_per_sentence": cands / args.sample, "segments_per_sentence": segs / args.sample,
        "candidates_per_position": cands / positions, "segments_per_position": segs / positions,
        "segments_per_position_hist": {str(k): seg_hist[k] for k in sorted(seg_hist)},
        "batch": cfg["batch"], "pool_bytes_old": old_b, "pool_bytes_new": new_b,
        # K2 writes the pool once and the Viterbi kernel reads it once
        "dram_bytes_per_step_old": 2 * old_b, "dram_bytes_per_step_new": 2 * new_b,
    }
    print(f"config {args.config}: {res['candidates_per_position']:.2f} candidates and {res['segments_per_position']:.2f} "
          f"segments per position; pool {old_b / 1e9:.2f} GB as records, {new_b / 1e9:.2f} GB as segments per batch of "
          f"{cfg['batch']} sentences")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
