#!/usr/bin/env python3
"""Small run of marginals, lattice and sampling together on the layout k_viterbi2<4> with sort_by_length 2 (eight
sentences per warp, dealt through Batch::order), for compute-sanitizer memcheck and racecheck, checked against the
restatements as tests/test_gpu_prob_layouts.py checks them: the ties adversarial dictionary (rows longer than one
staging pass, positions with more than 32 candidates), ignore_space on, whole batch and device-resident input.
Kernels: k_viterbi2<4>, k_marg_forward / k_marg_backward through Batch::order, k_lattice_*, k_sample_*.

    tools/run_sanitizer.sh layouts memcheck racecheck"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import adversarial as adv  # noqa: E402
import test_gpu_prob_layouts as t  # noqa: E402
from bounded_oracle import BoundedOracle  # noqa: E402
from test_gpu_marginals import adversarial_dicts  # noqa: E402

THETA = 0.01
d, dev, od = adversarial_dicts("ties")
bo = BoundedOracle(od, d.char_def, d.unk_def, True)
sents = adv.make_sentences(d, 40, seed=13, max_len=60) + ["", "   ", " a  "]
exp = t.Expected([t.sentence_expect(bo, s, THETA, i) for i, s in enumerate(sents)])
for device in (False, True):
    tok = t.make_tok(dev, True, THETA, kernel=1, lanes=4, sort=2)
    got = t.run(tok, sents, device=device)
    assert tok.describe()["last_viterbi"] == "k_viterbi2"
    t.check(got, exp, bo, sents, THETA, f"device={device}")
print(f"layouts probe ok: {len(sents)} sentences, {len(exp.nodes)} nodes, worst {t.mo.F32_ULPS['worst']} ulps")
