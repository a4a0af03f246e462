"""The segment-encoded candidate pool at its limits, on every route, against the oracle (tests/segment_fixtures.py;
tests/test_segment_model.py shows on the CPU that each fixture reaches its edge):

* far ends: end slots more than 32 767 (and 65 534) away from the slot before them, reached through move segments;
* big sources: postings lists and an unk.def category of 2^16 candidates or more, split into several segments;
* crowded positions: 7 / 8 / 9, G - 1 / G / G + 1 (G = 4, 8, 16, 32) and more than 33 segments;
* a batch with more segments than candidates, whose pool the segments alone overflow.

Tokens and offsets are byte-identical to the C oracle (counters and connection-id counts too), bounded calls to
BoundedOracle; marginals and lattice nodes match their restatements, and token_probs / node_probs are bit-identical
across routes."""
import numpy as np
import pytest

import adversarial as adv
import lattice_oracle as lo
import marginal_oracle as mo
import segment_fixtures as sf
import vibrato_b200 as vb
from bounded_oracle import BoundedOracle
from oracle import vibrato_oracle as vo
from test_gpu_marginals import d2h, shard_devices
from test_gpu_viterbi_routes import expected_route

pytestmark = pytest.mark.gpu
LANES = (4, 8, 16, 32)
THETA = 0.01


@pytest.fixture(scope="module")
def dic():
    lex, matrix, char_def, unk_def, user, long_word = sf.make_dictionary()
    dev = vb.SystemDictionaryBuilder.from_readers(lex, matrix, char_def, unk_def).reset_user_lexicon_from_reader(user)
    od = vo.OracleDictionary(lex, matrix, char_def, unk_def).set_user_csv(user)
    return dev, od, unk_def, long_word


def assert_tokens(off, toks, e_off, e_toks, what=""):
    np.testing.assert_array_equal(off, e_off, err_msg=str(what))
    assert len(toks) == len(e_toks), what
    for name in vb.TOKEN_DTYPE.names:
        np.testing.assert_array_equal(toks[name], e_toks[name], err_msg=f"{name} {what}")


def device_call(tok, sents, bounds=None):
    """tokenize_batch_device: (tok_off, tokens) copied back."""
    import torch
    utf8, off = adv.pack(sents)
    d_utf8 = torch.from_numpy(utf8.copy() if len(utf8) else np.zeros(1, np.uint8)).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    kw = {}
    if bounds is not None:
        bo, bnd = vb.Tokenizer.pack_bounds(bounds)
        d_bo = torch.from_numpy(bo.astype(np.int64)).cuda()
        d_bnd = torch.from_numpy(bnd.astype(np.int32) if len(bnd) else np.zeros(1, np.int32)).cuda()
        kw = dict(d_bnd_offsets=d_bo.data_ptr(), d_bnd=d_bnd.data_ptr(), n_bnd=len(bnd))
    torch.cuda.synchronize()
    a, b, n = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), len(sents), len(utf8), **kw)
    return d2h(a, len(sents) + 1, np.uint64), d2h(b, n, vb.TOKEN_DTYPE)


def every_route(dev, od, sents, long_sentence, isp=False, mgl=0):
    """viterbi_kernel 0 / 1 / 2 x lanes, counted, connid_counting, chunked (a sentence per chunk), compact records,
    device-resident input and a two-entry multi-device tokenizer (shard_devices), all against the C oracle."""
    utf8, off = adv.pack(sents)
    e_off, e_toks, e_cnt = od.tokenize_batch(utf8, off, isp, mgl, n_threads=8, want_counters=True)
    tok = vb.Tokenizer.new(dev).ignore_space(isp).max_grouping_len(mgl)
    for kernel in (0, 1, 2):
        for lanes in LANES:
            tok.set_option("viterbi_kernel", kernel)
            tok.set_option("lanes_per_sentence", lanes)
            res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
            assert tok.describe()["last_viterbi"] == expected_route(kernel, long_sentence=long_sentence), (kernel, lanes)
            assert_tokens(res.tok_offsets, res.tokens, e_off, e_toks, (kernel, lanes))
    tok.set_option("viterbi_kernel", 1)
    tok.set_counting(True)
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
    assert tok.describe()["last_viterbi"] == "k_viterbi"
    assert_tokens(res.tok_offsets, res.tokens, e_off, e_toks, "counted")
    np.testing.assert_array_equal(tok.last_counters(), e_cnt)
    tok.set_counting(False)
    tok.init_connid_counter()
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
    assert_tokens(res.tok_offsets, res.tokens, e_off, e_toks, "connid")
    lid, rid = tok.connid_counts()
    olid, orid = od.connid_counts(utf8, off, isp, mgl, n_threads=8)
    np.testing.assert_array_equal(lid, olid)
    np.testing.assert_array_equal(rid, orid)
    chunked = vb.Tokenizer.new(dev).ignore_space(isp).max_grouping_len(mgl)
    chunked.set_option("chunk_sentences", 1)
    res = chunked.tokenize_batch(utf8=utf8, byte_offsets=off)
    assert chunked.describe()["last_viterbi"] == expected_route(1, long_sentence=long_sentence)
    assert_tokens(res.tok_offsets, res.tokens, e_off, e_toks, "chunked")
    compact = vb.Tokenizer.new(dev).ignore_space(isp).max_grouping_len(mgl).compact_tokens(True)
    res = compact.tokenize_batch(utf8=utf8, byte_offsets=off)
    assert_tokens(res.tok_offsets, res.tokens, e_off, e_toks, "compact")
    assert_tokens(*device_call(vb.Tokenizer.new(dev).ignore_space(isp).max_grouping_len(mgl), sents), e_off, e_toks, "device")
    multi = vb.Tokenizer.new(dev, devices=shard_devices(2)).ignore_space(isp).max_grouping_len(mgl)
    res = multi.tokenize_batch(utf8=utf8, byte_offsets=off)
    assert_tokens(res.tok_offsets, res.tokens, e_off, e_toks, "multi")


@pytest.mark.parametrize("isp,mgl", [(False, 0), (True, 0), (False, 40000)])
def test_far_ends(dic, isp, mgl):
    """Sentences of 98 303 / 150 000 characters and 40 000-space runs: every positive end-slot delta up to the run's
    length and every negative one down to -(g - 1), some groups over max_grouping_len and some under it.  The batch
    holds sentences over 16 000 characters, so viterbi_kernel 1 must take the unpruned twin."""
    dev, od, _, long_word = dic
    every_route(dev, od, sf.far_sentences(long_word), True, isp, mgl)


def test_crowded_positions_and_big_sources(dic):
    """Crowded positions and 2^16-candidate sources, all sentences within 16 000 characters: the pruned k_viterbi2
    sees them with every lanes_per_sentence."""
    dev, od, _, _ = dic
    sents = sf.crowd_sentences() + sf.big_sentences() + sf.crowd_sentences()[::-1]
    every_route(dev, od, sents, False)
    every_route(dev, od, sf.crowd_sentences(), False, True)


def test_small_batch(dic):
    """Batches within 16 KiB and 131 072 candidates take k_small_batch; a 65 537-homograph word next to the
    70 000-entry unknown character outgrows its pool and falls back to the usual route with the same tokens."""
    dev, od, _, _ = dic
    tok = vb.Tokenizer.new(dev)
    tok.small_batch(64)
    for sents, small in ([sf.crowd_sentences(), True], [["kb"], True], [["lb", "blb"], False], [["lb"], True],
                         [["mb", "ab"], True], [["nb"], True], [["bnb"], True], [["bXb"], True], [["mbXb"], False],
                         [["mb", "bXb"], False]):
        utf8, off = adv.pack(sents)
        e_off, e_toks, _ = od.tokenize_batch(utf8, off)
        res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
        assert (tok.describe()["last_viterbi"] == "k_small_batch") == small, sents
        assert_tokens(res.tok_offsets, res.tokens, e_off, e_toks, sents)


def test_segments_outnumber_candidates(dic):
    """A pool sized for the candidates but not the segments: the segments alone overflow it, the batch is re-run
    with the size it needed, and a second call fits the learned estimate.  Whole batch with connection-id counting,
    and the chunked pipeline.  The engine reports no retry count, so nothing here shows that the retry ran: the
    regime rests on tests/test_segment_model.py, whose want_cand restates the pool sizing of ensure_workspace.  A
    change to that sizing (slack on the segment buffer, say) must be carried into want_cand, or this becomes a plain
    run."""
    dev, od, _, _ = dic
    sents = sf.OUTNUMBER_SENTENCES
    utf8, off = adv.pack(sents)
    e_off, e_toks, _ = od.tokenize_batch(utf8, off)
    olid, orid = od.connid_counts(utf8, off)
    for chunk in (0, 1):
        tok = vb.Tokenizer.new(dev)
        tok.set_option("pool_estimate_permille", sf.OUTNUMBER_PERMILLE)
        tok.set_option("chunk_sentences", chunk)
        tok.init_connid_counter()
        for call in range(2):
            res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
            assert_tokens(res.tok_offsets, res.tokens, e_off, e_toks, (chunk, call))
            lid, rid = tok.connid_counts()
            np.testing.assert_array_equal(lid, (call + 1) * olid)
            np.testing.assert_array_equal(rid, (call + 1) * orid)


def test_bounded(dic):
    """Boundaries that clip a group to exactly 32 767 / 32 768 characters and a crowded position to 8 / 9
    segments, against BoundedOracle, on every Viterbi kernel, the chunked pipeline, device-resident input and,
    within 16 KiB, k_small_batch."""
    dev, od, unk_def, _ = dic
    bo = BoundedOracle(od, sf.CHAR_DEF, unk_def)
    sents = [sf.CLIP_SENTENCE, sf.CLIP_SENTENCE, sf.CROWD_CLIP_SENTENCE, sf.CROWD_CLIP_SENTENCE] + sf.crowd_sentences()
    bounds = [list(b) for b in sf.CLIP_BOUNDS + sf.CROWD_CLIP_BOUNDS] + [[min(3, len(s))] for s in sf.crowd_sentences()]
    e_off, e_toks = bo.tokenize_batch([s.encode() for s in sents], bounds)
    utf8, off = adv.pack(sents)
    tok = vb.Tokenizer.new(dev)
    for kernel in (0, 1, 2):
        for lanes in (4, 32):
            tok.set_option("viterbi_kernel", kernel)
            tok.set_option("lanes_per_sentence", lanes)
            res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds)
            assert tok.describe()["last_viterbi"] == expected_route(kernel, long_sentence=True)
            assert_tokens(res.tok_offsets, res.tokens, e_off, e_toks, (kernel, lanes))
    chunked = vb.Tokenizer.new(dev)
    chunked.set_option("chunk_sentences", 1)
    res = chunked.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds)
    assert_tokens(res.tok_offsets, res.tokens, e_off, e_toks, "chunked")
    assert_tokens(*device_call(vb.Tokenizer.new(dev), sents, bounds), e_off, e_toks, "device")
    small_sents, small_bounds = sents[2:], bounds[2:]
    s_off, s_toks = bo.tokenize_batch([s.encode() for s in small_sents], small_bounds)
    small = vb.Tokenizer.new(dev)
    small.small_batch(64)
    u8, o = adv.pack(small_sents)
    res = small.tokenize_batch(utf8=u8, byte_offsets=o, boundaries=small_bounds)
    assert small.describe()["last_viterbi"] == "k_small_batch"
    assert_tokens(res.tok_offsets, res.tokens, s_off, s_toks, "small")


MARG_ROUTES = ("whole", "chunked", "compact", "device", "viterbi0", "unpruned")


def marg_lattice_run(dev, route, sents, bounds=None):
    """(tok_off, tokens, token_probs, node_off, nodes, links, node_probs) with marginals and lattice on."""
    tok = vb.Tokenizer.new(dev)
    if route == "chunked":
        tok.set_option("chunk_sentences", 1)
    if route == "compact":
        tok.compact_tokens(True)
    if route == "viterbi0":
        tok.set_option("viterbi_kernel", 0)
    if route == "unpruned":
        tok.set_option("viterbi_kernel", 2)
    tok.marginals(THETA)
    tok.lattice(True)
    if route == "device":
        a, b = device_call(tok, sents, bounds)
        tp = d2h(tok.last_device_marginals()[0], len(b), np.float32)
        no, nd, nl, npb, nn = tok.last_device_lattice()
        return (a, b, tp, d2h(no, len(sents) + 1, np.uint64), d2h(nd, nn, vb.TOKEN_DTYPE), d2h(nl, nn, vb.LINK_DTYPE),
                d2h(npb, nn, np.float32))
    utf8, off = adv.pack(sents)
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds)
    return (res.tok_offsets.copy(), res.tokens.copy(), res.token_probs.copy(), res.node_offsets.copy(), res.nodes.copy(),
            res.node_links.copy(), res.node_probs.copy())


def check_routes_identical(dev, sents, bounds=None):
    """Every route gives the same tokens, nodes and links, and bit-identical token_probs / node_probs."""
    base = marg_lattice_run(dev, "whole", sents, bounds)
    best = (base[5]["flags"] & vb.NODE_BEST) != 0
    assert base[4][best].tobytes() == base[1].tobytes() and base[6][best].tobytes() == base[2].tobytes()
    for route in MARG_ROUTES[1:]:
        got = marg_lattice_run(dev, route, sents, bounds)
        assert_tokens(got[0], got[1], base[0], base[1], route)  # compact records come back expanded
        for i in (2, 3, 4, 5, 6):
            assert got[i].tobytes() == base[i].tobytes(), (route, i)
    return base


def test_marginals_and_lattice(dic):
    """One sentence per fixture through the marginal and lattice restatements (nodes and links exact, probabilities
    within the tolerance of tests/test_gpu_marginals.py), then token_probs / node_probs bit-identical across routes,
    also on the far-end batch, which is too long for the restatements."""
    dev, od, unk_def, long_word = dic
    bo = BoundedOracle(od, sf.CHAR_DEF, unk_def)
    sents = ["Z" * 33000, sf.crowd_sentence(33), sf.crowd_sentence(9), "mb", "nb", "bnb", "bXb", ""]
    bounds = [[32768], [], [2], [], [], [], [], []]
    for b in (None, bounds):
        got = check_routes_identical(dev, sents, b)
        enc = [s.encode() for s in sents]
        e_off, e_toks = bo.tokenize_batch(enc, b)
        assert_tokens(got[0], got[1], e_off, e_toks, b)
        e_tp, _ = mo.batch_marginals(bo, enc, THETA, b)
        n_off, nodes, links, probs = lo.batch_lattice(bo, enc, b, THETA)
        np.testing.assert_array_equal(got[3], n_off)
        assert got[4].tobytes() == nodes.tobytes() and got[5].tobytes() == links.tobytes()
        mo.assert_f32_close(got[2], e_tp, what="token_probs")
        mo.assert_f32_close(got[6], probs, what="node_probs")
    far = sf.far_sentences(long_word)
    got = check_routes_identical(dev, far)
    e_off, e_toks, _ = od.tokenize_batch(*adv.pack(far))
    assert_tokens(got[0], got[1], e_off, e_toks, "far")
