"""Required tokens at the limits of their device code, against the span oracle (fixtures: tests/span_fixtures.py;
tests/test_span_limits_model.py shows on the CPU that each one reaches its edge):

* filtered 2^16-word lists and the 70 000-entry unknown category: runs split at 0xFFFF, a kept record past u16,
  tens of thousands of runs at one start (re-walked straight into the pool), the unknown fallback;
* crowded span starts of 3 ... 33 segments (kMaxSegs +- 1, G - 1 / G / G + 1 of every lanes_per_sentence);
* quoted features (`"a,b"`, `""`, empty and trailing fields, 256 fields) against a pattern battery;
* spans of 32 766 ... 98 303 characters, also behind a 40 000-space run with ignore_space;
* 31 ... 200 spans per sentence, a span over 150 000 characters, and lists whose 33rd span is invalid.

With the lattice on, the nodes from each span's start to its end carry exactly the oracle's word_idx list, in order,
so a wrong pattern decision or a mis-decoded segment shows even off the best path.  Tokens are byte-identical to
SpanOracle on every route; marginals, lattice, near-best margins and samples match their restatements."""
import time

import numpy as np
import pytest

import lattice_oracle as lo
import margin_oracle as mgo
import marginal_oracle as mo
import segment_fixtures as sf
import span_fixtures as spf
import test_gpu_sampling as tgs
import vibrato_b200 as vb
from oracle import vibrato_oracle as vo
from span_oracle import Constraints, SpanOracle
from test_gpu_spans import assert_guarantee
from test_gpu_spans import run as spans_run

pytestmark = pytest.mark.gpu
THETA = 0.01
N, SEED = 3, 20261017  # samples per sentence, Philox seed
LANES, SORTS = (4, 8, 16, 32), (0, 1, 2)
ROUTES = ("whole", "chunked", "compact", "overflow", "small", "device")
timings = {}
draws = {"ambiguous": 0, "of": 0}


@pytest.fixture(scope="module")
def big():
    lex, matrix, char_def, unk_def, user, long_word = spf.make_dictionary()
    dev = vb.SystemDictionaryBuilder.from_readers(lex, matrix, char_def, unk_def).reset_user_lexicon_from_reader(user)
    od = vo.OracleDictionary(lex, matrix, char_def, unk_def).set_user_csv(user)
    return dev, {isp: SpanOracle(od, char_def, unk_def, isp) for isp in (False, True)}, long_word


@pytest.fixture(scope="module")
def quoted():
    lex, matrix, char_def, unk_def = spf.make_quoted()
    dev = vb.SystemDictionaryBuilder.from_readers(lex, matrix, char_def, unk_def)
    od = vo.OracleDictionary(lex, matrix, char_def, unk_def)
    return dev, SpanOracle(od, char_def, unk_def)


class Expected:
    """The oracle's tokens of a batch, and per sentence and span the word_idx list of the nodes from its start to its
    end, in lattice order."""

    def __init__(self, so, sents, spans):
        self.cons = [Constraints((), tuple(sp)) for sp in spans]
        self.enc = [s.encode() for s in sents]
        self.off, self.toks = so.tokenize_batch(self.enc, self.cons)
        self.toks = self.toks.astype(vb.TOKEN_DTYPE)
        self.span_words, self.n_cand = [], []
        for b, c in zip(self.enc, self.cons):
            trace = []
            _, _, c2b = so.lattice(b, c, trace=trace)
            b2c = {x: i for i, x in enumerate(c2b)}
            self.span_words.append([[w for _, sw, ew, w in trace if (sw, ew) == (b2c[a], b2c[e])] for a, e, *_ in c.spans])
            self.n_cand.append(len(trace))


def joined(parts):
    """One Expected of the batches of `parts` (Expected objects) in a row."""
    out = Expected.__new__(Expected)
    for name in ("cons", "enc", "span_words", "n_cand"):
        setattr(out, name, [x for e in parts for x in getattr(e, name)])
    per = np.concatenate([np.diff(e.off.astype(np.int64)) for e in parts])
    out.off = np.zeros(len(per) + 1, dtype=np.uint64)
    out.off[1:] = np.cumsum(per)
    out.toks = np.concatenate([e.toks for e in parts])
    return out


def overflows(exp):
    """Does the batch hold more candidates than the pool that pool_estimate_permille = 1 gives it (the smallest one,
    segment_fixtures.want_cand restating engine.cu's sizing)?  The oracle's count is a lower bound of the device's:
    K2 also gives candidates to positions no path reaches.  The engine reports no retry count, so this is what shows
    that the overflow route re-runs the batch."""
    return sum(exp.n_cand) > sf.want_cand(sum(len(b) for b in exp.enc), 1)


# 70 000 BIG candidates at one start: more than the smallest pool on its own
FILLER = (["Xb"], [[(0, 1)]])


def overflow_batch(so, exp, sents, spans, filler):
    """The batch the overflow route runs: `filler` in front where the dictionary has the BIG category, else the batch
    repeated, until it overflows the smallest pool."""
    if filler and not overflows(exp):
        exp, sents, spans = joined([Expected(so, *FILLER), exp]), FILLER[0] + sents, FILLER[1] + spans
    n, b = sum(exp.n_cand), sum(len(x) for x in exp.enc)
    assert n > 0
    k = 1
    while k * n <= sf.want_cand(k * b, 1):
        k += 1
    exp = joined([exp] * k)
    assert overflows(exp)
    return exp, sents * k, spans * k


def make_tok(dev, route="whole", isp=False, chunk=3):
    tok = vb.Tokenizer.new(dev).ignore_space(isp)
    if route == "chunked":
        tok.set_option("chunk_sentences", chunk)
    if route == "compact":
        tok.compact_tokens(True)
    if route == "overflow":  # the smallest pool, which the batch (overflow_batch) outgrows: the batch runs again
        tok.set_option("pool_estimate_permille", 1)
    if route == "small":
        tok.small_batch(64)
    return tok


def check_route(dev, route, exp, sents, spans, isp=False, chunk=3, lattice=True):
    """Tokens byte-identical to the oracle's on `route`; with the lattice on, every span's nodes as well."""
    if route == "overflow":
        assert overflows(exp)
    tok = make_tok(dev, route, isp, chunk)
    if route == "device":
        off, toks = spans_run(tok, "device", sents, spans, [[] for _ in sents])
    else:
        tok.lattice(lattice)
        res = tok.tokenize_batch(sents, spans=spans)
        if route == "small":  # k_small_batch steps aside for spans
            assert tok.describe()["last_viterbi"] != "k_small_batch"
        off, toks = res.tok_offsets, res.tokens
        if lattice:
            check_span_nodes(res.node_offsets, res.nodes, exp, spans, route)
    np.testing.assert_array_equal(off, exp.off, err_msg=route)
    assert toks.tobytes() == exp.toks.tobytes(), route
    assert_guarantee(sents, spans, off, toks)


def check_span_nodes(node_off, nodes, exp, spans, what=""):
    for i, sp in enumerate(spans):
        nd = nodes[int(node_off[i]):int(node_off[i + 1])]
        for (a, e, *_), want in zip(sp, exp.span_words[i]):
            got = nd["word_idx"][(nd["start_byte"] == a) & (nd["end_byte"] == e)]
            assert got.tolist() == want, (what, i, a, e, len(got), len(want))


def every_route(dev, so, sents, spans, isp=False, chunk=3, lattice=True, filler=True):
    """filler: the dictionary has the BIG category (FILLER), which the overflow route puts in front of a small batch."""
    t0 = time.perf_counter()
    exp = Expected(so, sents, spans)
    big = overflow_batch(so, exp, sents, spans, filler)
    t1 = time.perf_counter()
    for route in ROUTES:
        if route == "overflow":
            check_route(dev, route, *big, isp, chunk, lattice)
        else:
            check_route(dev, route, exp, sents, spans, isp, chunk, lattice)
    return t1 - t0, time.perf_counter() - t1


def test_big_lists_and_crowded_starts(big):
    """Every selector pattern on the 65 535 / 65 536 / 65 537-word lists and the 70 000 BIG entries, at a sentence's
    start and after a word, and the crowded starts of 3 ... 33 segments, on every route."""
    dev, sos, _ = big
    sents, spans = spf.big_spans(spf.BIG_SPAN_CASES)
    cs, csp = spf.crowd_cases()
    timings["big lists + crowded (oracle, GPU)"] = every_route(dev, sos[False], sents + cs, spans + csp)


def test_quoted_features(quoted):
    dev, so = quoted
    sents, spans = spf.quoted_cases()
    exp = Expected(so, sents, spans)
    ids = [wid for wid, end in so.od.common_prefix(spf.QUOTED_SURFACE) if end == 2]
    for k, (pat, want) in enumerate(spf.QUOTED_PATTERNS.items()):  # the first sentence of each pattern: "ab"
        words = exp.span_words[3 * k][0]
        if want:
            assert words == [ids[i] for i in want], pat
        else:
            assert [w & 0xFFFF for w in words] == [(so.unk_off[2] + i) & 0xFFFF for i in spf.QUOTED_UNK_PATTERNS[pat]]
    big = overflow_batch(so, exp, sents, spans, False)
    t0 = time.perf_counter()
    for route in ROUTES:
        if route == "overflow":
            check_route(dev, route, *big)
        else:
            check_route(dev, route, exp, sents, spans)
    timings["quoted (GPU)"] = time.perf_counter() - t0


@pytest.mark.parametrize("isp", [False, True])
def test_far_spans(big, isp):
    """Spans of 32 766 ... 98 303 characters from the start of a `Z` run and from the middle of an ALPHA run, the long
    user word spanned with and without its feature; with ignore_space, the same behind 40 000 spaces."""
    dev, sos, long_word = big
    sents, spans, isp_sents, isp_spans = spf.far_cases(long_word)
    if isp:
        sents, spans = isp_sents, isp_spans
    timings[f"far spans isp={int(isp)} (oracle, GPU)"] = every_route(dev, sos[isp], sents, spans, isp, chunk=1)


def test_many_spans(big):
    """31 ... 200 spans per sentence, chunk-edge ends, a span over 150 000 characters; then lists whose 33rd span is
    invalid are refused, and the same tokenizer gives the right bytes on the next call."""
    dev, sos, _ = big
    so = sos[False]
    sents, spans = spf.many_cases()
    timings["many spans (oracle, GPU)"] = every_route(dev, so, sents, spans, lattice=False)
    exp = Expected(so, sents[:4], spans[:4])
    for route in ("whole", "chunked"):
        tok = make_tok(dev, route)
        for s, sp, bnd in spf.refused_cases():
            with pytest.raises(vb.VibratoError, match="spans") as e:
                tok.tokenize_batch(sents[:4] + [s], spans=spans[:4] + [sp], boundaries=[[]] * 4 + [bnd])
            assert e.value.kind == "InvalidArgument"
            res = tok.tokenize_batch(sents[:4], spans=spans[:4])
            np.testing.assert_array_equal(res.tok_offsets, exp.off)
            assert res.tokens.tobytes() == exp.toks.tobytes()


def test_quadratic_start(big):
    """Tens of thousands of segments at one span start (every second record of `m`, every third of `n`, every second
    BIG entry), whose candidates cand_at finds by walking from the first segment: on the whole batch route only,
    timed.  The warm-up call with the same batch outgrows the first pool and runs again; the timed call fits the
    estimate it learned, so it times one pass."""
    dev, sos, _ = big
    sents, spans = spf.big_spans(spf.QUADRATIC_CASES)
    exp = Expected(sos[False], sents, spans)
    tok = vb.Tokenizer.new(dev).lattice(True)
    tok.tokenize_batch(sents, spans=spans)  # warm up
    t0 = time.perf_counter()
    res = tok.tokenize_batch(sents, spans=spans)
    timings["quadratic start (GPU, one call)"] = time.perf_counter() - t0
    np.testing.assert_array_equal(res.tok_offsets, exp.off)
    assert res.tokens.tobytes() == exp.toks.tobytes()
    check_span_nodes(res.node_offsets, res.nodes, exp, spans, "quadratic")


# --- downstream outputs over span lattices ------------------------------------------------------------------------
def downstream_tok(dev, kernel=1, lanes=16, sort=0, margin=None):
    tok = vb.Tokenizer.new(dev).marginals(THETA).lattice(True, margin=margin).sampling(N, THETA, SEED)
    tok.set_option("viterbi_kernel", kernel)
    tok.set_option("lanes_per_sentence", lanes)
    tok.set_option("sort_by_length", sort)
    return tok


def downstream_run(tok, sents, spans):
    res = tok.tokenize_batch(sents, spans=spans)
    res.close()
    out = (res.tok_offsets, res.tokens, res.token_probs, res.path_probs, res.node_offsets, res.nodes, res.node_links,
           res.node_probs, res.sample_offsets, res.samples)
    return out + ((res.node_margins,) if res.node_margins is not None else ())


def check_downstream(got, so, exp, sents):
    """Tokens, nodes and links exact, probabilities within 2 float32 ulps, samples byte-identical up to ambiguous
    draws."""
    tok_off, toks, tp, pp, node_off, nodes, links, node_probs, s_off, samples = got[:10]
    np.testing.assert_array_equal(tok_off, exp.off)
    assert toks.tobytes() == exp.toks.tobytes()
    e_tp, e_pp = mo.batch_marginals(so, exp.enc, THETA, exp.cons)
    mo.assert_f32_close(tp, e_tp, what="token_probs")
    mo.assert_f32_close(pp, e_pp, what="path_probs")
    e_off, e_nodes, e_links, e_probs = lo.batch_lattice(so, exp.enc, exp.cons, THETA)
    np.testing.assert_array_equal(node_off, e_off)
    assert nodes.tobytes() == e_nodes.astype(vb.TOKEN_DTYPE).tobytes()
    assert links.tobytes() == e_links.astype(vb.LINK_DTYPE).tobytes()
    mo.assert_f32_close(node_probs, e_probs, what="node_probs")
    check_span_nodes(node_off, nodes, exp, [c.spans for c in exp.cons])
    before = tgs.ambiguous["samples"]
    tgs.check_parity(so, sents, (s_off, samples), N, THETA, SEED, bounds=exp.cons)
    draws["ambiguous"] += tgs.ambiguous["samples"] - before
    draws["of"] += len(sents) * N


def check_margins(got, so, exp, D):
    e_off, e_nodes, e_links, e_margins, e_probs = mgo.batch_pruned_lattice(so, exp.enc, D, exp.cons, THETA)
    node_off, nodes, links, node_probs, margins = got[4], got[5], got[6], got[7], got[10]
    np.testing.assert_array_equal(node_off, e_off)
    assert nodes.tobytes() == e_nodes.astype(vb.TOKEN_DTYPE).tobytes()
    assert links.tobytes() == e_links.astype(vb.LINK_DTYPE).tobytes()
    assert margins.tobytes() == e_margins.tobytes()
    mo.assert_f32_close(node_probs, e_probs, what=f"margin {D} node_probs")


def downstream_batch(big, quoted, fixture):
    if fixture == "quoted":
        return quoted[0], quoted[1], *spf.quoted_cases()
    dev, sos, _ = big
    # a run split at 0xFFFF, a run that starts past u16, the best record past u16 after a word and the BIG entry
    # past u16; the crowded starts
    bs, bsp = spf.big_spans([("all", "lb", 0), ("hi", "mb", 0), ("best", "bnb", 1), ("best", "Xb", 0)])
    cs, csp = spf.crowd_cases()
    return dev, sos[False], bs + cs, bsp + csp


@pytest.mark.parametrize("fixture", ["big", "quoted"])
def test_downstream(big, quoted, fixture):
    """Marginals, lattice, near-best margins (0 and MAX_MARGIN) and samples over the span lattices of the filtered
    big lists and the crowded starts, and of the quoted battery."""
    dev, so, sents, spans = downstream_batch(big, quoted, fixture)
    t0 = time.perf_counter()
    exp = Expected(so, sents, spans)
    check_downstream(downstream_run(downstream_tok(dev), sents, spans), so, exp, sents)
    for D in (0, mgo.MAX_MARGIN):
        got = downstream_run(downstream_tok(dev, margin=D), sents, spans)
        check_margins(got, so, exp, D)
    timings[f"downstream {fixture}"] = time.perf_counter() - t0


@pytest.mark.parametrize("fixture", ["crowded", "quoted"])
def test_layout_matrix(big, quoted, fixture):
    """viterbi_kernel 0 / 1 / 2 x lanes_per_sentence 4 / 8 / 16 / 32 x sort_by_length 0 / 1 / 2 with marginals, lattice
    and sampling on: every output byte-identical to the lanes 16 / sort 0 run, which matches the restatements."""
    if fixture == "crowded":
        dev, so = big[0], big[1][False]
        sents, spans = spf.crowd_cases()
    else:
        dev, so = quoted
        sents, spans = spf.quoted_cases()
    t0 = time.perf_counter()
    ref = None
    for kernel in (0, 1, 2):
        for lanes in (16,) + tuple(x for x in LANES if x != 16):
            for sort in SORTS:
                got = downstream_run(downstream_tok(dev, kernel, lanes, sort), sents, spans)
                if ref is None:
                    check_downstream(got, so, Expected(so, sents, spans), sents)
                    ref = got
                for k, (a, b) in enumerate(zip(got, ref)):
                    assert a.tobytes() == b.tobytes(), (kernel, lanes, sort, k)
    timings[f"layouts {fixture}"] = time.perf_counter() - t0


def test_report():
    """Prints the worst float32 distance, the ambiguous draws and the seconds each test above took (run in the same
    session)."""
    print(f"span limits: worst distance from the restatements = {mo.F32_ULPS['worst']} float32 ulps")
    print(f"  samples with an ambiguous draw: {draws['ambiguous']} of {draws['of']}")
    for k, v in timings.items():
        print(f"  {k}: " + (", ".join(f"{x:.1f}" for x in v) if isinstance(v, tuple) else f"{v:.2f}") + " s")
