"""Segmentation uncertainty on the GPU (option "uncertainty"): entropy and log_path_prob within 1e-9 of the restatement
(tests/uncertainty_oracle.py), boundary probabilities within 2 float32 ulps of its float64 values, on the golden and
adversarial dictionaries, wrapping costs and rows of 2^16 entries; the exact cases (single path, empty and no-path
sentences, a sentence past path_prob's underflow); bounded and span calls; every route byte for byte against the
whole-batch call; every other output unchanged at levels 0, 1 and 2; errors, replay and the accessors."""
import math

import numpy as np
import pytest

import adversarial as adv
import marginal_oracle as mo
import segment_fixtures as sf
import uncertainty_oracle as uo
import vibrato_b200 as vb
from bounded_oracle import BoundedOracle
from oracle import vibrato_oracle as vo
from span_oracle import Constraints, SpanOracle
from test_gpu_marginals import adversarial_dicts, d2h, golden_dicts, golden_sents, shard_devices

pytestmark = pytest.mark.gpu
THETA = 0.01


def make(d, route="whole", level=2, isp=False, mgl=0, theta=THETA, chunk=64, lanes=None, sort=None, lattice=False,
         margin=None, samples=0):
    if route.startswith("multi"):
        tok = vb.Tokenizer.new(d, devices=shard_devices(2))
    else:
        tok = vb.Tokenizer.new(d)
    tok.ignore_space(isp).max_grouping_len(mgl)
    if route == "chunked":
        tok.set_option("chunk_sentences", chunk)
    if route == "compact":
        tok.compact_tokens(True)
    if route == "small":
        tok.small_batch(65536)
    if route == "viterbi0":
        tok.set_option("viterbi_kernel", 0)
    if route == "unpruned":
        tok.set_option("viterbi_kernel", 2)
    if lanes is not None:
        tok.set_option("lanes_per_sentence", lanes)
    if sort is not None:
        tok.set_option("sort_by_length", sort)
    if lattice or margin is not None:
        tok.lattice(True, margin=margin)
    if samples:
        tok.sampling(samples, theta, seed=5)
    tok.marginals(theta)
    if level:
        tok.uncertainty(True, boundary_probs=level >= 2)
    return tok


def run(tok, route, sents, bounds=None, spans=None):
    """dict of the call's outputs: ent, lpp, boff, bprob (None at level 1), tokens, token_probs, path_probs."""
    utf8, off = adv.pack(sents)
    if route in ("device", "multi_device"):
        import torch
        d_utf8 = torch.from_numpy(utf8.copy() if len(utf8) else np.zeros(1, np.uint8)).cuda()
        d_off = torch.from_numpy(off.astype(np.int64)).cuda()
        kw = {}
        if bounds is not None:
            bo, bnd = vb.Tokenizer.pack_bounds(bounds)
            d_bo = torch.from_numpy(bo.astype(np.int64)).cuda()
            d_bnd = torch.from_numpy(bnd.astype(np.int32) if len(bnd) else np.zeros(1, np.int32)).cuda()
            kw = dict(d_bnd_offsets=d_bo.data_ptr(), d_bnd=d_bnd.data_ptr(), n_bnd=len(bnd))
        torch.cuda.synchronize()
        _, b, n = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), len(sents), len(utf8), **kw)
        de, dl, dbo, dbp, npos = tok.last_device_uncertainty()
        ns = len(sents)
        tp, pp = tok.last_device_marginals()
        return dict(ent=d2h(de, ns, np.float64), lpp=d2h(dl, ns, np.float64),
                    boff=d2h(dbo, ns + 1, np.uint64) if dbo else None, bprob=d2h(dbp, npos, np.float32) if dbp else None,
                    tokens=d2h(b, n, vb.TOKEN_DTYPE), token_probs=d2h(tp, n, np.float32), path_probs=d2h(pp, ns, np.float32))
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds, spans=spans)
    if route == "small":
        assert tok.describe()["last_viterbi"] != "k_small_batch"
    res.close()
    return dict(ent=res.entropies, lpp=res.log_path_probs, boff=res.boundary_offsets, bprob=res.boundary_probs,
                tokens=res.tokens, token_probs=res.token_probs, path_probs=res.path_probs)


def close64(got, exp, tol=1e-9):
    got, exp = np.asarray(got, dtype=np.float64), np.asarray(exp, dtype=np.float64)
    assert got.shape == exp.shape
    inf = np.isinf(exp)
    assert np.array_equal(np.isinf(got), inf) and np.array_equal(got[inf], exp[inf])
    err = np.abs(got[~inf] - exp[~inf])
    ok = err <= tol * np.maximum(1.0, np.abs(exp[~inf]))
    assert ok.all(), (int(np.argmin(ok)), got[~inf][~ok][:3], exp[~inf][~ok][:3])


def check(bo, sents, got, theta=THETA, bounds=None, exp=None):
    exp = exp or uo.batch_uncertainty(bo, [s.encode() for s in sents], theta, bounds)
    e_ent, e_lpp, e_off, e_bnd = exp
    close64(got["ent"], e_ent)
    close64(got["lpp"], e_lpp)
    # path_prob is the float32 of exp(log_path_prob), to one ulp
    pp = np.exp(got["lpp"]).astype(np.float32)
    dist = np.abs(pp.view(np.int32).astype(np.int64) - got["path_probs"].view(np.int32).astype(np.int64))
    assert dist.max(initial=0) <= 1
    if got["bprob"] is not None:
        np.testing.assert_array_equal(got["boff"], e_off)
        mo.assert_f32_close(got["bprob"], e_bnd, ulps=2, what="boundary_probs")
    return exp


def test_golden(golden):
    sents = golden_sents(golden) + ["東京 都  ", "   ", ""]
    for user in (False, True):
        d, od, r = golden_dicts(golden, user)
        for isp, mgl in ((False, 0), (True, 0), (False, 3)):
            bo = BoundedOracle(od, r["char.def"], r["unk.def"], isp, mgl)
            for theta in (THETA, 0.001):
                check(bo, sents, run(make(d, isp=isp, mgl=mgl, theta=theta), "whole", sents), theta)


@pytest.mark.parametrize("family", list(adv.FAMILIES) + ["raw", "dual"])
def test_adversarial(family):
    """The matrix families and the "wrap" dictionaries (Raw and Dual connectors), whose costs run near +-2^31."""
    d, dev, od = adversarial_dicts(family)
    sents = adv.make_sentences(d, 40, seed=7, max_len=40) + [""]
    theta = 0.05 if family in adv.FAMILIES else 1e-7
    for isp in (False, True):
        bo = BoundedOracle(od, d.char_def, d.unk_def, isp)
        check(bo, sents, run(make(dev, isp=isp, theta=theta), "whole", sents), theta)


@pytest.mark.parametrize("w,c", [(-32768, -32768), (32767, 32767)])
def test_wrapping_path_costs(w, c):
    sents = ["a" * 3000, "a" * 7, "", " " + "a" * 2000 + "  "]
    for aa in (None, 0):
        files = adv.single_word_dictionary(w, c, with_aa=aa)
        dev = vb.SystemDictionaryBuilder.from_readers(*files)
        for isp in (False, True):
            bo = BoundedOracle(vo.OracleDictionary(*files), files[2], files[3], isp)
            exp = uo.batch_uncertainty(bo, [s.encode() for s in sents], 1e-4)
            for route in ("whole", "viterbi0", "unpruned"):
                check(bo, sents, run(make(dev, route, isp=isp, theta=1e-4), route, sents), 1e-4, exp=exp)


def test_big_rows():
    """Rows of 2^16 entries and more: the per-lane sums and the boundary rows past u16."""
    lex, matrix, char_def, unk_def, user, _ = sf.make_dictionary()
    dev = vb.SystemDictionaryBuilder.from_readers(lex, matrix, char_def, unk_def).reset_user_lexicon_from_reader(user)
    od = vo.OracleDictionary(lex, matrix, char_def, unk_def).set_user_csv(user)
    bo = BoundedOracle(od, char_def, unk_def)
    sents = sf.crowd_sentences() + sf.big_sentences()
    exp = uo.batch_uncertainty(bo, [s.encode() for s in sents], THETA)
    for route in ("whole", "unpruned"):
        check(bo, sents, run(make(dev, route), route, sents), exp=exp)


def zero_dict():
    z = adv.zero_dictionary()
    dev = vb.SystemDictionaryBuilder.from_readers(z.lex_csv, z.matrix, z.char_def, z.unk_def)
    return z, dev, BoundedOracle(vo.OracleDictionary(z.lex_csv, z.matrix, z.char_def, z.unk_def), z.char_def, z.unk_def)


def test_exact_cases(golden):
    """A single path gives 0.0 / 0.0 exactly; empty sentences (also across chunk edges) 0 / 0 / [1]; a sentence past
    path_prob's float32 underflow a finite log_path_prob equal to -ln T(n) and the restatement."""
    z, dev, bo = zero_dict()
    sents = ["b", "", "a" * 200, "aab", ""]
    got = run(make(dev), "whole", sents)
    assert got["ent"][0] == 0.0 and got["lpp"][0] == 0.0
    assert got["ent"][1] == 0.0 and got["lpp"][1] == 0.0
    assert got["path_probs"][2] == 0.0 and np.isfinite(got["lpp"][2]) and got["lpp"][2] < -103
    h, lpp = uo.exact_uncertainty(mo.Lattice(bo, b"a" * 200), 1)
    close64(got["ent"][2:3], [h], 1e-12)
    close64(got["lpp"][2:3], [lpp], 1e-12)
    check(bo, sents, got)
    bo_ = got["boff"]
    assert got["bprob"][int(bo_[1]):int(bo_[2])].tolist() == [1.0]
    # runs of empty sentences across chunk edges
    d, od, r = golden_dicts(golden, True)
    gbo = BoundedOracle(od, r["char.def"], r["unk.def"])
    sents = [""] * 150 + golden_sents(golden) * 20 + [""] * 130
    exp = uo.batch_uncertainty(gbo, [s.encode() for s in sents], THETA)
    for route in ("whole", "chunked", "device"):
        check(gbo, sents, run(make(d, route, chunk=100), route, sents), exp=exp)
    for route in ("whole", "device"):
        got = run(make(d, route), route, [])
        assert len(got["ent"]) == 0 and got["boff"].tolist() == [0] and len(got["bprob"]) == 0


def test_no_path(golden):
    """A span over hiragana, which the fixture's unk.def has no entry for: 0 / -inf / all zeros."""
    d, od, r = golden_dicts(golden, True)
    so = SpanOracle(od, r["char.def"], r["unk.def"])
    sents = ["ぬぬ京都", "京都東京都京都"]
    spans = [[(0, 6, None)], []]
    got = run(make(d), "whole", sents, spans=spans)
    assert got["ent"][0] == 0.0 and got["lpp"][0] == -math.inf
    assert got["bprob"][:5].tolist() == [0.0] * 5
    check(so, sents, got, bounds=[Constraints((), tuple(s)) for s in spans])


def test_bounds_and_spans(golden):
    """Required boundaries and span ends within 2 ulps of 1, span interiors exactly 0, and the restatement."""
    d, od, r = golden_dicts(golden, True)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    sents = ["京都東京都京都", "abcdefgh", "", "東京に行った。"]
    bounds = [[6, 12], [3], [], [9]]
    one = np.float32(1.0)
    for route in ("whole", "chunked", "device"):
        got = check(bo, sents, run(make(d, route, chunk=2), route, sents, bounds), bounds=bounds)
        g = run(make(d, route, chunk=2), route, sents, bounds)
        for i, (s, bl) in enumerate(zip(sents, bounds)):
            b0 = int(g["boff"][i])
            c2b = [len(s[:k].encode()) for k in range(len(s) + 1)]
            for bb in bl:
                v = g["bprob"][b0 + c2b.index(bb)]
                assert abs(int(np.float32(v).view(np.int32)) - int(one.view(np.int32))) <= 2, (s, bb, v)
    so = SpanOracle(od, r["char.def"], r["unk.def"])
    spans = [[(6, 15, None)], [(0, 3, None)], [], [(0, 6, "名詞")]]
    cons = [Constraints((), tuple(s)) for s in spans]
    g = run(make(d), "whole", sents, spans=spans)
    check(so, sents, g, bounds=cons)
    inside = {0: [3, 4], 1: [1, 2], 3: [1]}
    for i, ps in inside.items():
        b0 = int(g["boff"][i])
        assert all(g["bprob"][b0 + p] == 0.0 for p in ps)
    for i, end in ((0, 5), (1, 3), (3, 2)):
        v = g["bprob"][int(g["boff"][i]) + end]
        assert abs(int(np.float32(v).view(np.int32)) - int(one.view(np.int32))) <= 2


def same(a, b):
    for k in a:
        if a[k] is None or b[k] is None:
            assert a[k] is None and b[k] is None, k
        else:
            assert a[k].tobytes() == b[k].tobytes(), k


ROUTES = ["chunked", "device", "compact", "small", "viterbi0", "unpruned"]


def test_routes_byte_for_byte(golden):
    """Every route, chunk size, lanes / sort layout, and the lattice, near-best lattice and sampling on and off: the
    same bytes as the whole-batch call."""
    d, od, r = golden_dicts(golden, True)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    sents = golden_sents(golden) * 20 + [""] * 70 + ["東京 都  " * 9] * 5 + golden_sents(golden) * 10
    ref = run(make(d), "whole", sents)
    check(bo, sents, ref)
    ref.pop("tokens")
    for route in ROUTES:
        got = run(make(d, route), route, sents)
        got.pop("tokens")
        same(ref, got)
    for chunk in (16, 100, 1000):
        got = run(make(d, "chunked", chunk=chunk), "chunked", sents)
        got.pop("tokens")
        same(ref, got)
    for lanes in (4, 8, 16, 32):
        for sort in (0, 1, 2):
            for kernel in ("whole", "viterbi0"):
                got = run(make(d, kernel, lanes=lanes, sort=sort), kernel, sents)
                got.pop("tokens")
                same(ref, got)
    for kw in (dict(lattice=True), dict(margin=500), dict(samples=3), dict(lattice=True, samples=2)):
        for route in ("whole", "chunked", "device"):
            got = run(make(d, route, **kw), route, sents)
            got.pop("tokens")
            same(ref, got)
    # level 1: the same per-sentence values and no boundary arrays
    got = run(make(d, level=1), "whole", sents)
    assert got["bprob"] is None and got["boff"] is None
    assert got["ent"].tobytes() == ref["ent"].tobytes() and got["lpp"].tobytes() == ref["lpp"].tobytes()
    got = run(make(d, "device", level=1), "device", sents)
    assert got["bprob"] is None and got["ent"].tobytes() == ref["ent"].tobytes()


@pytest.mark.parametrize("route", ["multi", "multi_device"])
def test_multi_device(golden, route):
    d, od, r = golden_dicts(golden, True)
    sents = golden_sents(golden) * 40 + [""] * 70 + golden_sents(golden) * 30
    ref = run(make(d), "whole", sents)
    got = run(make(d, route), "device" if route == "multi_device" else "whole", sents)
    same(ref, got)


def test_other_outputs_unchanged(golden):
    """Tokens, marginals, lattice, margins, samples and text are byte-identical at levels 0, 1 and 2."""
    d, od, r = golden_dicts(golden, True)
    sents = golden_sents(golden) * 3
    utf8, off = adv.pack(sents)
    outs = []
    for level in (0, 1, 2):
        tok = vb.Tokenizer.new(d).marginals(THETA).sampling(2, THETA, seed=9).output_mode("mecab")
        tok.lattice(True, margin=3000)
        if level:
            tok.uncertainty(True, boundary_probs=level == 2)
        res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
        outs.append([res.tokens.tobytes(), res.token_probs.tobytes(), res.path_probs.tobytes(), res.samples.tobytes(),
                     res.nodes.tobytes(), res.node_links.tobytes(), res.node_probs.tobytes(),
                     res.node_margins.tobytes(), res.text()[1]])
        assert (res.entropies is None) == (level == 0) and (res.boundary_probs is None) == (level < 2)
    assert outs[0] == outs[1] == outs[2]
    for level in (0, 2):  # without the rest, and on the eager small-batch path
        tok = vb.Tokenizer.new(d).marginals(THETA)
        if level:
            tok.uncertainty(True, True)
        res = tok.tokenize_batch(["京都東京都京都", "", "に"])
        outs.append((res.tokens.tobytes(), res.token_probs.tobytes(), res.path_probs.tobytes()))
    assert outs[-1] == outs[-2]


def test_errors_replay_and_accessors(golden):
    d, od, r = golden_dicts(golden, True)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    tok = vb.Tokenizer.new(d)
    with pytest.raises(vb.VibratoError, match="marginals"):
        tok.uncertainty(True)
    with pytest.raises(vb.VibratoError, match="marginals"):
        tok.set_option("uncertainty", 2)
    tok.marginals(THETA)
    for bad in (-1, 3):
        with pytest.raises(vb.VibratoError, match="uncertainty must be"):
            tok.set_option("uncertainty", bad)
    tok.uncertainty(True, boundary_probs=True)
    with pytest.raises(vb.VibratoError, match="marginals"):
        tok.marginals(0)
    res = tok.tokenize_batch(["京都東京都京都", ""])
    assert res.sentence_boundary_probs(1).tolist() == [1.0]
    assert len(res.sentence_boundary_probs(0)) == 8
    tok.ignore_space(True)  # rebuilds the engine: the option is replayed
    res2 = tok.tokenize_batch(["京都東京都京都", ""])
    assert res2.entropies.tobytes() == res.entropies.tobytes()
    assert res2.boundary_probs.tobytes() == res.boundary_probs.tobytes()
    w = tok.new_worker()
    w.reset_sentence("京都東京都京都")
    w.tokenize()
    assert w.entropy() == float(res.entropies[0]) and w.log_path_prob() == float(res.log_path_probs[0])
    assert w.boundary_probs().tobytes() == res.sentence_boundary_probs(0).tobytes()
    w.reset_sentence("")
    w.tokenize()
    assert w.entropy() == 0.0 and w.log_path_prob() == 0.0 and w.boundary_probs().tolist() == [1.0]
    tok.uncertainty(True)  # level 1
    res = tok.tokenize_batch(["京都東京都京都"])
    assert res.boundary_probs is None and res.entropies is not None
    with pytest.raises(vb.VibratoError, match="boundary"):
        res.sentence_boundary_probs(0)
    w.reset_sentence("京都")
    w.tokenize()
    with pytest.raises(vb.VibratoError, match="boundary"):
        w.boundary_probs()
    tok.uncertainty(False)
    tok.marginals(0)  # allowed again
    res = tok.tokenize_batch(["京都"])
    assert res.entropies is None
    w.reset_sentence("京都")
    w.tokenize()
    with pytest.raises(vb.VibratoError, match="no uncertainty"):
        w.entropy()
    import torch
    x = torch.from_numpy(np.frombuffer("京都".encode(), np.uint8).copy()).cuda()
    o = torch.tensor([0, 6], dtype=torch.int64).cuda()
    plain = vb.Tokenizer.new(d).marginals(THETA)
    plain.tokenize_batch_device(x.data_ptr(), o.data_ptr(), 1, 6)
    with pytest.raises(vb.VibratoError, match="uncertainty"):
        plain.last_device_uncertainty()
    plain.uncertainty(True)
    plain.tokenize_batch_device(x.data_ptr(), o.data_ptr(), 1, 6)
    de, dl, dbo, dbp, npos = plain.last_device_uncertainty()
    assert de and dl and dbo == 0 and dbp == 0 and npos == 0
    e = uo.batch_uncertainty(bo, ["京都".encode()], THETA)
    close64(d2h(de, 1, np.float64), e[0])
