#!/usr/bin/env python3
"""Developer tool: cost of the device-side output stage (k_format_len / k_format_write) on the host path.
    python tools/format_probe.py [dict] [batch]"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import vibrato_b200 as vb  # noqa: E402
from vibrato_b200 import synth  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else "synth-unidic"
batch = int(sys.argv[2]) if len(sys.argv) > 2 else 1000000
sd = synth.make_dictionary(name)
utf8, off = synth.make_corpus(sd, batch, seed=20260925)
d = vb.SystemDictionaryBuilder.from_readers(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
tok = vb.Tokenizer.new(d)
h_utf8 = torch.from_numpy(utf8).pin_memory().numpy()
h_off = torch.from_numpy(off.astype(np.int64)).pin_memory().numpy().view(np.uint64)
tok.set_option("chunk_sentences", 0)  # the whole-batch route throughout (tools/output_bench.py compares the routes)
base = None
for mode in (None, "wakati", "mecab", "detail"):
    tok.output_mode(mode)
    nbytes = 0
    for _ in range(2):
        tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off).close()
    t = time.perf_counter()
    for _ in range(3):
        r = tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off)
        torch.cuda.synchronize()
        del r
    wall = (time.perf_counter() - t) / 3 * 1e3
    if mode is not None:
        r = tok.tokenize_batch(utf8=h_utf8, byte_offsets=h_off)
        nbytes = len(r.text()[1])
        del r
    base = wall if base is None else base
    extra = wall - base
    print(f"mode={str(mode):7s} host-path wall={wall:8.2f} ms  text={nbytes / 1e6:9.1f} MB  extra vs tokens only={extra:8.2f} ms"
          + (f"  ({nbytes / 1e9 / (extra * 1e-3):6.1f} GB/s of text incl. its D2H copy)" if mode and extra > 0 else ""), flush=True)
