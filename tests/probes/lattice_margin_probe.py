#!/usr/bin/env python3
"""Small run of the near-best lattice for compute-sanitizer memcheck, checked against the restatement
(tests/margin_oracle.py): whole batch, the chunked pipeline (empty sentences at chunk edges) and device-resident input,
with and without marginals (the R-only forward pass and the shared one), ignore_space on, then lattice text with %pb.
Kernels: k_marg_forward's R-only instantiation, k_margin_backward, k_lattice_count_margin, k_lattice_write<true>.

    tools/run_sanitizer.sh lattice_margin memcheck"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import adversarial as adv  # noqa: E402
import margin_oracle as mgo  # noqa: E402
import torch  # noqa: E402
import vibrato_b200 as vb  # noqa: E402
from bounded_oracle import BoundedOracle  # noqa: E402
from oracle import vibrato_oracle as vo  # noqa: E402

THETA = 0.01
D = 2000
g = json.load(open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8"))
r = g["resources"]
d = vb.SystemDictionaryBuilder.from_readers(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
bo = BoundedOracle(od, r["char.def"], r["unk.def"], True)
base = [c["input"] for c in g["tokenizer_cases"]] + ["京都東京都京都", "東京   都", "abc  ", "", " 東京"]


def d2h(ptr, n, dtype):
    from cuda.bindings import runtime as cudart
    host = np.empty(n, dtype=dtype)
    if n:
        (err,) = cudart.cudaMemcpy(host.ctypes.data, ptr, host.nbytes, cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost)
        assert int(err) == 0
    return host


for theta in (0, THETA):
    for route in ("whole", "chunked", "device"):
        tok = vb.Tokenizer.new(d).ignore_space(True).marginals(theta).lattice(True, margin=D)
        sents = base
        if route == "chunked":
            tok.set_option("chunk_sentences", 64)
            sents = base * 20 + [""] * 70 + base * 10
        e_off, e_nodes, e_links, e_margins, _ = mgo.batch_pruned_lattice(bo, [s.encode() for s in sents], D)
        utf8, off = adv.pack(sents)
        if route == "device":
            t = [torch.from_numpy(x).cuda() for x in (utf8.copy(), off.astype(np.int64))]
            torch.cuda.synchronize()
            tok.tokenize_batch_device(t[0].data_ptr(), t[1].data_ptr(), len(sents), len(utf8))
            no, nd, nl, _, nn = tok.last_device_lattice()
            got = (d2h(no, len(sents) + 1, np.uint64), d2h(nd, nn, vb.TOKEN_DTYPE), d2h(nl, nn, vb.LINK_DTYPE),
                   d2h(tok.last_device_lattice_margins(), nn, np.int64))
        else:
            res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
            got = (res.node_offsets, res.nodes, res.node_links, res.node_margins)
        assert np.array_equal(got[0], e_off) and got[1].tobytes() == e_nodes.tobytes()
        assert got[2].tobytes() == e_links.tobytes() and got[3].tobytes() == e_margins.tobytes()

tok = vb.Tokenizer.new(d).lattice(True, text=True, margin=0).output_format("%pb%m\n")
_, text = tok.tokenize_batch(base).text()
assert text.count(b"*") > 0
print("lattice margin probe ok")
