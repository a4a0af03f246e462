"""Marginals, lattice and samples on every layout of the Viterbi stage (K3), against the restatements and the exact
marginals.

k_marg_forward numbers every candidate's lattice entry again (BOS first, then positions in order, then candidates
in candidate order), the lattice lists the nodes in that order and the sampling walks index the same rows: all three
rely on K3 inserting nodes in exactly that order, whichever kernel runs, however many lanes a sentence gets
(k_viterbi2<G> pools the candidates of 32 / G sentences per warp) and in whatever order the sentences are dealt
(sort_by_length 1 and 2 map warps and walks through Batch::order).  Each node folds its terms in row order, so no
probability may change by a single bit from one layout to another.

* the layout matrix: viterbi_kernel 0 / 1 / 2 x lanes_per_sentence 4 / 8 / 16 / 32 x sort_by_length 0 / 1 / 2,
  plus a chunked, a counted, a device-resident and a bounded run, on the golden and adversarial dictionaries;
* k_backtrack<true, kBackTile> (batches of at least 256 sentences per SM) against k_backtrack<true, 32>;
* exact path counts (tests/marginal_oracle.exact_marginals) on sentences of up to 20 000 characters with more than
  10^308 paths, and exact power-of-two weights."""
import functools
import math
import time

import numpy as np
import pytest

import adversarial as adv
import lattice_oracle as lo
import marginal_oracle as mo
import sampling_oracle as so
import vibrato_b200 as vb
from bounded_oracle import BoundedOracle
from oracle import vibrato_oracle as vo
from test_gpu_marginals import adversarial_dicts, d2h, golden_dicts, golden_sents
from test_gpu_sampling import check_parity
from test_gpu_viterbi_routes import LANES, SORTS, expected_route

pytestmark = pytest.mark.gpu
N, SEED = 3, 20261017  # samples per sentence, Philox seed
DICTS = ("golden", "ties", "flat_columns", "extreme", "raw", "dual")
PRED_CAP = 32  # kPredCap: k_viterbi2 stages a row's predecessors in passes of 32
timings = {}
ambiguous = {}  # (dictionary, ignore_space) -> samples of the matrix compared only up to an ambiguous draw


def golden_corpus(golden, n_sent, seed, max_len=200):
    """Sentences of 0-`max_len` characters (log-uniform) cut from the golden cases and space runs."""
    pieces = [s for s in golden_sents(golden) if s] + [" ", "   "]
    rng = np.random.default_rng([seed, 5])
    lens = np.floor(np.exp(rng.uniform(0, np.log(max_len + 1), n_sent))).astype(np.int64)
    out = []
    for n in lens.tolist():
        s = ""
        while len(s) < n:
            s += pieces[int(rng.integers(0, len(pieces)))]
        out.append(s[:n])
    return out


def sentence_expect(bo, s, theta, i, bounds=()):
    """(token_probs, path_prob, nodes, links, node_probs, samples, mo.Lattice or None) of sentence i from one
    restated lattice."""
    b = s.encode()
    nodes, links, _ = lo.sentence_lattice(bo, b, bounds)
    if not b:
        return [], 1.0, nodes, links, [], so.sentence_samples(bo, b, N, theta, SEED, i), None
    lat = mo.Lattice(bo, b, bounds)
    prob, pp, _ = mo.marginals(lat, theta)
    fw = so.forward(lat, theta)
    samples = []
    for j in range(N):
        path, amb = so.walk(lat, fw, theta, SEED, i, j)
        samples.append((so.records(lat, path), path, amb))
    return [prob[n] for n in lat.best_path()], pp, nodes, links, [prob[n] for n in lat.nodes[1:]], samples, lat


class Expected:
    """The restatements' outputs of a batch, flat like BatchResult's."""

    def __init__(self, per):
        self.per = per
        self.tp = np.array([x for p in per for x in p[0]], dtype=np.float64)
        self.pp = np.array([p[1] for p in per], dtype=np.float64)
        counts = [len(p[2]) for p in per]
        self.node_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64)
        self.nodes = np.concatenate([p[2] for p in per])
        self.links = np.concatenate([p[3] for p in per])
        self.node_probs = np.array([x for p in per for x in p[4]], dtype=np.float64)
        best = (self.links["flags"] & lo.NODE_BEST) != 0
        self.tokens = self.nodes[best]  # the tokens are the lattice's best-path nodes (tests/test_gpu_lattice.py)
        bc = np.array([int(np.count_nonzero((p[3]["flags"] & lo.NODE_BEST) != 0)) for p in per], dtype=np.uint64)
        self.tok_off = np.concatenate([[0], np.cumsum(bc)]).astype(np.uint64)
        self.samples = [p[5] for p in per]


@functools.lru_cache(maxsize=None)
def setup(name, isp):
    """(device dictionary, oracle, sentences, theta, connector, Expected) of one dictionary and ignore_space."""
    import json
    import os
    if name == "golden":
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vibrato_fixture.json"),
                  encoding="utf-8") as f:
            golden = json.load(f)
        dev, od, r = golden_dicts(golden, True)
        bo = BoundedOracle(od, r["char.def"], r["unk.def"], isp)
        sents = golden_corpus(golden, 240, seed=3)
        connector, theta = "matrix", 0.01
    else:
        d, dev, od = adversarial_dicts(name)
        bo = BoundedOracle(od, d.char_def, d.unk_def, isp)
        sents = adv.make_sentences(d, 240, seed=13, max_len=200)
        connector = name if name in ("raw", "dual") else "matrix"
        theta = 0.01 if connector == "matrix" else 1e-6  # the wrap family's costs are near +-2^31
    sents += ["", " ", "   ", "", " a  ", "  "]
    t0 = time.perf_counter()
    per = [sentence_expect(bo, s, theta, i) for i, s in enumerate(sents)]
    lats = [p[6] for p in per if p[6] is not None]
    if name != "golden":  # rows past one staging pass and positions past one warp of candidates are in the batch
        assert max(len(row) for lat in lats for row in lat.ends) > PRED_CAP
        assert max(len(v) for lat in lats for v in lat.succ.values()) > 32
    exp = Expected(per)
    timings[f"restate {name} isp={int(isp)}"] = time.perf_counter() - t0
    ambiguous[(name, isp)] = sum(amb is not None for smp in exp.samples for _, _, amb in smp)
    return dev, bo, sents, theta, connector, exp


def make_tok(dev, isp, theta, kernel=1, lanes=16, sort=0, chunk=0, counted=False):
    tok = vb.Tokenizer.new(dev).ignore_space(isp).marginals(theta).lattice(True).sampling(N, theta, SEED)
    tok.set_option("viterbi_kernel", kernel)
    tok.set_option("lanes_per_sentence", lanes)
    tok.set_option("sort_by_length", sort)
    tok.set_option("chunk_sentences", chunk)
    tok.set_counting(counted)
    return tok


def run(tok, sents, device=False, bounds=None):
    """(tok_off, tokens, token_probs, path_probs, node_off, nodes, links, node_probs, sample_off, samples)"""
    utf8, off = adv.pack(sents)
    if device:
        import torch
        d_utf8 = torch.from_numpy(utf8.copy() if len(utf8) else np.zeros(1, np.uint8)).cuda()
        d_off = torch.from_numpy(off.astype(np.int64)).cuda()
        torch.cuda.synchronize()
        a, b, n = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), len(sents), len(utf8))
        tp, pp = tok.last_device_marginals()
        no, nd, nl, npb, nn = tok.last_device_lattice()
        so_ptr, s_ptr, ns = tok.last_device_samples()
        return (d2h(a, len(sents) + 1, np.uint64), d2h(b, n, vb.TOKEN_DTYPE), d2h(tp, n, np.float32),
                d2h(pp, len(sents), np.float32), d2h(no, len(sents) + 1, np.uint64), d2h(nd, nn, vb.TOKEN_DTYPE),
                d2h(nl, nn, vb.LINK_DTYPE), d2h(npb, nn, np.float32), d2h(so_ptr, len(sents) * N + 1, np.uint64),
                d2h(s_ptr, ns, vb.TOKEN_DTYPE))
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds)
    res.close()
    return (res.tok_offsets, res.tokens, res.token_probs, res.path_probs, res.node_offsets, res.nodes, res.node_links,
            res.node_probs, res.sample_offsets, res.samples)


def check(got, exp, bo, sents, theta, what):
    tok_off, toks, tp, pp, node_off, nodes, links, node_probs, s_off, samples = got
    np.testing.assert_array_equal(tok_off, exp.tok_off, err_msg=what)
    assert toks.tobytes() == exp.tokens.tobytes(), what
    mo.assert_f32_close(tp, exp.tp, what=f"{what} token_probs")
    mo.assert_f32_close(pp, exp.pp, what=f"{what} path_probs")
    np.testing.assert_array_equal(node_off, exp.node_off, err_msg=what)
    assert nodes.tobytes() == exp.nodes.tobytes(), what
    assert links.tobytes() == exp.links.tobytes(), what
    mo.assert_f32_close(node_probs, exp.node_probs, what=f"{what} node_probs")
    best = (links["flags"] & vb.NODE_BEST) != 0
    assert node_probs[best].tobytes() == tp.tobytes(), what
    check_parity(bo, sents, (s_off, samples), N, theta, SEED, expected=exp.samples)


def same_bits(got, ref, what):
    """Every output, probabilities and samples included, is byte-identical to the reference layout's."""
    for k, (a, b) in enumerate(zip(got, ref)):
        assert a.tobytes() == b.tobytes(), (what, k)


@pytest.mark.parametrize("ignore_space", [False, True])
@pytest.mark.parametrize("name", DICTS)
def test_layout_matrix(name, ignore_space):
    """viterbi_kernel x lanes_per_sentence x sort_by_length, then a chunked, a counted, a device-resident and a bounded
    run: tokens, lattice and samples exact, probabilities within 2 float32 steps of the restatement and bit-identical
    to lanes 16 / sort 0."""
    dev, bo, sents, theta, connector, exp = setup(name, ignore_space)
    t0 = time.perf_counter()
    kernels = (0, 1, 2)
    ref = None
    for kernel in kernels:
        for lanes in (16,) + tuple(x for x in LANES if x != 16):
            for sort in SORTS:
                what = f"kernel {kernel} lanes {lanes} sort {sort}"
                tok = make_tok(dev, ignore_space, theta, kernel, lanes, sort)
                got = run(tok, sents)
                assert tok.describe()["last_viterbi"] == expected_route(kernel, connector=connector), what
                check(got, exp, bo, sents, theta, what)
                if ref is None:
                    assert (kernel, lanes, sort) == (0, 16, 0)
                    ref = got
                same_bits(got, ref, what)
    extra = (("chunked", dict(lanes=32, sort=1, chunk=100), False),
             ("counted", dict(lanes=8, sort=2, counted=True), False),
             ("device", dict(lanes=4, sort=2), True))
    for what, kw, device in extra:
        tok = make_tok(dev, ignore_space, theta, **kw)
        got = run(tok, sents, device=device)
        assert tok.describe()["last_viterbi"] == expected_route(1, counted=what == "counted", connector=connector), what
        check(got, exp, bo, sents, theta, what)
        same_bits(got, ref, what)
    # bounded: a boundary in the middle of every fifth sentence where the lattice keeps a path to EOS (without one the
    # restatements have no value); the others keep their expected values
    bounds = []
    for i, s in enumerate(sents):
        bnd = [len(s[:len(s) // 2].encode())] if i % 5 == 0 and len(s) > 1 else []
        if bnd:
            ends, (eos_row, _), _ = bo.lattice(s.encode(), bnd)
            bnd = bnd if ends[eos_row] else []
        bounds.append(bnd)
    assert sum(map(bool, bounds)) >= len(sents) // 10
    per = [sentence_expect(bo, s, theta, i, tuple(bounds[i])) if bounds[i] else exp.per[i] for i, s in enumerate(sents)]
    bexp = Expected(per)
    tok = make_tok(dev, ignore_space, theta, lanes=4, sort=1)
    got = run(tok, sents, bounds=bounds)
    assert tok.describe()["last_viterbi"] == expected_route(1, connector=connector)
    check(got, bexp, bo, sents, theta, "bounded")
    ref_b = run(make_tok(dev, ignore_space, theta), sents, bounds=bounds)
    same_bits(got, ref_b, "bounded")
    timings[f"layouts {name} isp={int(ignore_space)}"] = time.perf_counter() - t0


@pytest.mark.parametrize("n_sent", [40000, 40255])
def test_large_back_tiles(n_sent):
    """Batches of at least 256 sentences per SM take k_backtrack<true, 256>: token_probs and path_probs as the
    restatement says, and bit-identical to the same batch in chunks of 1 000 sentences, which take
    k_backtrack<true, 32>; on the whole-batch, compact and device-resident routes, sentences sorted or not."""
    import torch
    t0 = time.perf_counter()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert n_sent >= 256 * sms and 1000 < 256 * sms
    d, dev, od = adversarial_dicts("ties")
    bo = BoundedOracle(od, d.char_def, d.unk_def)
    theta = 0.01
    distinct = adv.make_sentences(d, 97, seed=21, max_len=80)
    sents = [distinct[i % len(distinct)] for i in range(n_sent)]
    ref = [mo.sentence_marginals(bo, s.encode(), theta) for s in distinct]
    e_tp = np.array([x for i in range(n_sent) for x in ref[i % len(distinct)][0]], dtype=np.float64)
    e_pp = np.array([ref[i % len(distinct)][1] for i in range(n_sent)], dtype=np.float64)
    for sort in (0, 1):
        base = vb.Tokenizer.new(dev).marginals(theta)
        base.set_option("sort_by_length", sort)
        base.set_option("chunk_sentences", 1000)
        utf8, off = adv.pack(sents)
        small = base.tokenize_batch(utf8=utf8, byte_offsets=off)
        for route in ("whole", "compact", "device"):
            what = f"{route} sort {sort}"
            tok = vb.Tokenizer.new(dev).marginals(theta)
            tok.set_option("sort_by_length", sort)
            if route == "compact":
                tok.compact_tokens(True)
            if route == "device":
                d_utf8, d_off = torch.from_numpy(utf8.copy()).cuda(), torch.from_numpy(off.astype(np.int64)).cuda()
                torch.cuda.synchronize()
                a, b, n = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), n_sent, len(utf8))
                tp_ptr, pp_ptr = tok.last_device_marginals()
                tok_off, toks = d2h(a, n_sent + 1, np.uint64), d2h(b, n, vb.TOKEN_DTYPE)
                tp, pp = d2h(tp_ptr, n, np.float32), d2h(pp_ptr, n_sent, np.float32)
            else:
                res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
                tok_off, toks, tp, pp = res.tok_offsets, res.tokens, res.token_probs, res.path_probs
            np.testing.assert_array_equal(tok_off, small.tok_offsets, err_msg=what)
            if route != "compact":
                assert toks.tobytes() == small.tokens.tobytes(), what
            mo.assert_f32_close(tp, e_tp, what=f"{what} token_probs")
            mo.assert_f32_close(pp, e_pp, what=f"{what} path_probs")
            assert tp.tobytes() == small.token_probs.tobytes(), what
            assert pp.tobytes() == small.path_probs.tobytes(), what
    timings[f"large back tiles {n_sent}"] = time.perf_counter() - t0


def exact_pair(d):
    dev = vb.SystemDictionaryBuilder.from_readers(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    if d.user_csv:
        dev.reset_user_lexicon_from_reader(d.user_csv)
        od.set_user_csv(d.user_csv)
    return dev, BoundedOracle(od, d.char_def, d.unk_def)


def exact_expect(bo, sents, unit, bits):
    """(token_probs, path_probs, node_probs) from exact_marginals, flat like BatchResult's."""
    tp, pp, npb = [], [], []
    for s in sents:
        lat = mo.Lattice(bo, s.encode())
        prob, p = mo.exact_marginals(lat, unit, bits)
        tp += [prob[n] for n in lat.best_path()]
        npb += [prob[n] for n in lat.nodes[1:]]
        pp.append(p)
    return tuple(np.array(x, dtype=np.float64) for x in (tp, pp, npb))


def check_exact(dev, sents, exp, thetas, route):
    outs = []
    for theta in thetas:
        tok = vb.Tokenizer.new(dev).marginals(theta).lattice(True)
        res = tok.tokenize_batch(sents)
        assert tok.describe()["last_viterbi"] == route
        mo.assert_f32_close(res.token_probs, exp[0], what=f"theta {theta} token_probs")
        mo.assert_f32_close(res.path_probs, exp[1], what=f"theta {theta} path_probs")
        mo.assert_f32_close(res.node_probs, exp[2], what=f"theta {theta} node_probs")
        # underflow where the exact value underflows: float32 subnormals as they are, 0 where it rounds to 0
        np.testing.assert_array_equal(res.path_probs == 0, exp[1].astype(np.float32) == 0)
        outs.append((res.token_probs.tobytes(), res.path_probs.tobytes(), res.node_probs.tobytes()))
    assert all(o == outs[0] for o in outs), "the marginals of a zero-cost lattice depend on theta"


@pytest.mark.parametrize("long", [False, True])
def test_exact_path_counts(long):
    """Zero-cost dictionary, sentences of n `a`: T(n) paths (tribonacci, 10^5292 at n = 20 000), every marginal a
    ratio of path counts.  Within 2 float32 steps of the exact value, and bit-identical for theta 1e-6, 0.01 and 50.
    Sentences of more than 16 000 characters take the unpruned twin of k_viterbi2."""
    t0 = time.perf_counter()
    dev, bo = exact_pair(adv.zero_dictionary())
    lengths = (16001, 20000) if long else (1, 31, 33, 160, 512, 1000, 4000)
    sents = ["a" * n for n in lengths] + ([] if long else ["", "ab" * 60 + "bbb", "aabba a"])
    exp = exact_expect(bo, sents, 1, None)
    assert (exp[1][-1] if long else exp[1][lengths.index(4000)]) == 0.0  # fewer than 1 / 10^308: underflows
    check_exact(dev, sents, exp, (1e-6, 0.01, 50.0), expected_route(1, long_sentence=long))
    timings[f"exact zero long={int(long)}"] = time.perf_counter() - t0


def test_exact_pow2():
    """Costs that are multiples of 64 across i16 at theta = ln 2 / 64: every path weight a power of two.  Within 2
    float32 steps of the exact marginals (256-bit sums: tests/marginal_oracle.exact_marginals)."""
    t0 = time.perf_counter()
    d = adv.make_dictionary("pow2")
    dev, bo = exact_pair(d)
    sents = adv.make_sentences(d, 160, seed=6, max_len=200)
    sents += [("".join(sents) * 20)[:n] for n in (512, 1000, 4000)]
    exp = exact_expect(bo, sents, adv.POW2_UNIT, 256)
    check_exact(dev, sents, exp, (math.log(2) / adv.POW2_UNIT,), "k_viterbi2")
    timings["exact pow2"] = time.perf_counter() - t0


def test_report():
    """Prints the worst float32 distance and the seconds each test above took (run in the same session)."""
    print(f"prob layouts: worst distance from the reference = {mo.F32_ULPS['worst']} float32 ulps")
    print(f"  samples with an ambiguous draw (per sentence and sample, each layout): {sum(ambiguous.values())} of "
          f"{sum(len(setup(*k)[2]) * N for k in ambiguous)}")
    for k, v in timings.items():
        print(f"  {k}: {v:.1f} s")
