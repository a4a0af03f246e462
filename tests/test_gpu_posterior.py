"""Posterior decoding on the GPU (Tokenizer.posterior): bit for bit against the restatement (tests/posterior_oracle.py)
fed the device's own node marginals, on the golden, adversarial (Matrix / Raw / Dual), synth, wrapping-cost and
2^16-entry-row lattices; against the restatement's own float64 marginals; the guarantees of include/vibrato_b200.h
(a lattice path, the fold maximum, best-path records byte for byte); every route byte for byte; every other output
unchanged; posterior text; edge cases; errors, replay and the accessors."""
import math

import numpy as np
import pytest

import adversarial as adv
import marginal_oracle as mo
import posterior_oracle as po
import segment_fixtures as sf
import vibrato_b200 as vb
from bounded_oracle import BoundedOracle
from oracle import vibrato_oracle as vo
from span_oracle import Constraints, SpanOracle
from test_gpu_marginals import adversarial_dicts, d2h, golden_dicts, golden_sents, shard_devices, shard_devices_arg
from vibrato_b200 import synth
from vibrato_b200._native import check as vb_check, lib as vb_lib

pytestmark = pytest.mark.gpu
THETA = 0.01


def make(d, route="whole", gamma=1.0, isp=False, mgl=0, theta=THETA, chunk=64, lanes=None, sort=None, lattice=False,
         samples=0, unc=0, text=False):
    tok = vb.Tokenizer.new(d, devices=shard_devices(2)) if route.startswith("multi") else vb.Tokenizer.new(d)
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
    if lattice:
        tok.lattice(True)
    tok.marginals(theta)
    if samples:
        tok.sampling(samples, theta, seed=5)
    if unc:
        tok.uncertainty(True, boundary_probs=unc >= 2)
    if gamma is not None:
        tok.posterior(gamma, text=text)
    return tok


def run(tok, route, sents, bounds=None, spans=None):
    """dict of the call's outputs: poff, ptok, pprob, pgain, tokens, token_probs (and the lattice's when it is on)."""
    utf8, off = adv.pack(sents)
    ns = len(sents)
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
        _, b, n = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), ns, len(utf8), **kw)
        do, dt, dp, dg, npt = tok.last_device_posterior()
        tp, _ = tok.last_device_marginals()
        return dict(poff=d2h(do, ns + 1, np.uint64), ptok=d2h(dt, npt, vb.TOKEN_DTYPE), pprob=d2h(dp, npt, np.float32),
                    pgain=d2h(dg, ns, np.float64), tokens=d2h(b, n, vb.TOKEN_DTYPE), token_probs=d2h(tp, n, np.float32))
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds, spans=spans)
    if route == "small":
        assert tok.describe()["last_viterbi"] != "k_small_batch"
    res.close()
    out = dict(poff=res.posterior_offsets, ptok=res.posterior_tokens, pprob=res.posterior_probs,
               pgain=res.posterior_gains, tokens=res.tokens, token_probs=res.token_probs)
    if res.nodes is not None:
        out.update(node_off=res.node_offsets, node_probs=res.node_probs)
    if route == "compact":
        out.pop("tokens")
    return out


def lattice_of(bo, sent, cons):
    return mo.Lattice(bo, sent.encode(), cons if cons is not None else ())


def check_exact(bo, sents, got, gamma, cons=None):
    """Bit for bit against the restatement fed the device's own node_probs (the lattice must be on).  Returns the
    number of non-empty sentences with a path."""
    poff, nodeoff = got["poff"], got["node_off"]
    checked = 0
    for i, s in enumerate(sents):
        a, b = int(poff[i]), int(poff[i + 1])
        c = cons[i] if cons is not None else None
        if not s:
            assert a == b and got["pgain"][i] == 0.0
            continue
        lat = lattice_of(bo, s, c)
        order = [(e, k) for e in range(1, len(lat.ends)) for k in range(len(lat.ends[e]))]
        nprob = got["node_probs"][int(nodeoff[i]):int(nodeoff[i + 1])]
        assert len(nprob) == len(order), s
        p = dict(zip(order, nprob))
        if not lat.ends[lat.eos_row]:
            assert a == b and got["pgain"][i] == -math.inf
            continue
        path, v = po.sweep(lat, p, gamma)
        rec = po.records(lat, path)
        assert got["ptok"][a:b].tobytes() == rec.tobytes(), (s, got["ptok"][a:b], rec)
        assert got["pprob"][a:b].tobytes() == np.array([p[n] for n in path], dtype=np.float32).tobytes()
        assert got["pgain"][i] == v and v == po.fold(gamma + 1.0, p, path), (s, got["pgain"][i], v)
        checked += 1
    return checked


def check_float64(bo, sents, got, gamma, theta, cons=None):
    """Against the restatement's own float64 marginals: gains to 1e-6 relative, paths equal unless its two best folds
    are within 1e-6.  Returns the number of such near ties."""
    near = 0
    for i, s in enumerate(sents):
        if not s:
            continue
        lat = lattice_of(bo, s, cons[i] if cons is not None else None)
        if not lat.ends[lat.eos_row]:
            continue
        p = po.node_probs(lat, theta)
        path, v = po.sweep(lat, p, gamma)
        g = float(got["pgain"][i])
        assert abs(g - v) <= 1e-6 * max(1.0, abs(v)), (s, g, v)
        a, b = int(got["poff"][i]), int(got["poff"][i + 1])
        if got["ptok"][a:b].tobytes() != po.records(lat, path).tobytes():
            V, second = _two_best(lat, p, gamma)
            assert V - second <= 1e-6 * max(1.0, abs(V)), s
            near += 1
    return near


def _two_best(lat, p, gamma):
    """The two largest folds over every path (enumeration); where there are too many paths to enumerate, the sweep's
    value and -inf, so that a differing path there fails."""
    try:
        best, second, _ = po.brute_force(lat, p, gamma)
        return best, second
    except RuntimeError:
        return po.sweep(lat, p, gamma)[1], -math.inf


def report(where, near):
    print(f"{where}: {near} sentence(s) whose path differs from the float64 restatement's at a near tie")


def test_golden_exact(golden):
    sents = golden_sents(golden) + ["東京 都  ", "   ", "", "京都" * 40]
    checked = near = 0
    for user in (False, True):
        d, od, r = golden_dicts(golden, user)
        for isp, mgl in ((False, 0), (True, 0), (False, 3)):
            bo = BoundedOracle(od, r["char.def"], r["unk.def"], isp, mgl)
            for gamma in (0.0, 1.0, 8.0):
                got = run(make(d, gamma=gamma, isp=isp, mgl=mgl, lattice=True), "whole", sents)
                checked += check_exact(bo, sents, got, gamma)
                near += check_float64(bo, sents, got, gamma, THETA)
    assert checked > 50
    report("golden", near)


@pytest.mark.parametrize("family", list(adv.FAMILIES) + ["raw", "dual"])
def test_adversarial_exact(family):
    d, dev, od = adversarial_dicts(family)
    sents = adv.make_sentences(d, 40, seed=7, max_len=40) + [""]
    theta = 0.05 if family in adv.FAMILIES else 1e-7
    near = 0
    for isp in (False, True):
        bo = BoundedOracle(od, d.char_def, d.unk_def, isp)
        for gamma in (0.0, 1.0, 8.0):
            got = run(make(dev, gamma=gamma, isp=isp, theta=theta, lattice=True), "whole", sents)
            assert check_exact(bo, sents, got, gamma) > 20
            near += check_float64(bo, sents, got, gamma, theta)
    report(family, near)


def test_synth_exact():
    sd = synth.make_dictionary("synth-small")
    d = vb.SystemDictionaryBuilder.from_readers(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
    od = vo.OracleDictionary(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
    ucsv = synth.make_user_csv(sd, 200)
    d.reset_user_lexicon_from_reader(ucsv)
    od.set_user_csv(ucsv)
    utf8, off = synth.make_corpus(sd, 60, seed=11, log_uniform=(1, 40), unk_frac=0.15, space_frac=0.03, user_csv=ucsv,
                                  user_frac=0.05)
    sents = [bytes(utf8[int(off[i]):int(off[i + 1])]).decode() for i in range(len(off) - 1)]
    bo = BoundedOracle(od, sd.char_def, sd.unk_def, True, 24)
    for gamma in (0.0, 1.0, 8.0):
        got = run(make(d, gamma=gamma, isp=True, mgl=24, theta=0.0005, lattice=True), "whole", sents)
        assert check_exact(bo, sents, got, gamma) > 40


@pytest.mark.parametrize("w,c", [(-32768, -32768), (32767, 32767)])
def test_wrapping_path_costs(w, c):
    """Prefix costs in the tokenizer's wrapping i32 arithmetic, on long sentences whose costs pass +-2^31."""
    sents = ["a" * 3000, "a" * 7, "", " " + "a" * 2000 + "  "]
    for aa in (None, 0):
        files = adv.single_word_dictionary(w, c, with_aa=aa)
        dev = vb.SystemDictionaryBuilder.from_readers(*files)
        for isp in (False, True):
            bo = BoundedOracle(vo.OracleDictionary(*files), files[2], files[3], isp)
            for route in ("whole", "viterbi0", "unpruned"):
                got = run(make(dev, route, isp=isp, theta=1e-4, lattice=True), route, sents)
                check_exact(bo, sents, got, 1.0)


def test_big_rows():
    """Rows of 2^16 entries and more: the warp argmax over long rows, and predecessors past the u16 min_idx."""
    lex, matrix, char_def, unk_def, user, _ = sf.make_dictionary()
    dev = vb.SystemDictionaryBuilder.from_readers(lex, matrix, char_def, unk_def).reset_user_lexicon_from_reader(user)
    od = vo.OracleDictionary(lex, matrix, char_def, unk_def).set_user_csv(user)
    bo = BoundedOracle(od, char_def, unk_def)
    sents = sf.crowd_sentences() + sf.big_sentences()
    for route in ("whole", "unpruned"):
        got = run(make(dev, route, lattice=True), route, sents)
        assert check_exact(bo, sents, got, 1.0) >= 1


def test_guarantees(golden):
    """1: a BOS -> EOS path with the required boundaries and every span's token; 2: the gain is the fold, at least
    the best path's; 3: best-path nodes give the tokens' records and probabilities byte for byte."""
    d, od, r = golden_dicts(golden, True)
    so = SpanOracle(od, r["char.def"], r["unk.def"])
    sents = ["京都東京都京都", "abcdefgh", "", "東京に行った。", "京都東京都京都"]
    spans = [[(6, 15, None)], [(0, 3, None)], [], [(0, 6, "名詞")], [(0, 6, None), (6, 15, None), (15, 21, None)]]
    cons = [Constraints((), tuple(s)) for s in spans]
    for gamma in (0.0, 1.0, 8.0):
        got = run(make(d, gamma=gamma, lattice=True), "whole", sents, spans=spans)
        check_exact(so, sents, got, gamma, cons)
        for i, s in enumerate(sents):
            a, b = int(got["poff"][i]), int(got["poff"][i + 1])
            toks = got["ptok"][a:b]
            ends = {int(t["end_byte"]) for t in toks}
            assert all(e in ends for _, e, _ in spans[i]), (s, toks)
            assert all(any(int(t["start_byte"]) == st and int(t["end_byte"]) == e for t in toks) for st, e, _ in spans[i])
            if s:
                lat = lattice_of(so, s, cons[i])
                order = [(e, k) for e in range(1, len(lat.ends)) for k in range(len(lat.ends[e]))]
                p = dict(zip(order, got["node_probs"][int(got["node_off"][i]):int(got["node_off"][i + 1])]))
                assert got["pgain"][i] >= po.fold(gamma + 1.0, p, lat.best_path())
        # the forced alignment has one path: its records and probabilities are the tokens'
        res = make(d, gamma=gamma).tokenize_batch(sents, spans=spans)
        toff = res.tok_offsets
        i = 4
        assert (res.tokens[int(toff[i]):int(toff[i + 1])].tobytes() ==
                got["ptok"][int(got["poff"][i]):int(got["poff"][i + 1])].tobytes())
        assert (res.token_probs[int(toff[i]):int(toff[i + 1])].tobytes() ==
                got["pprob"][int(got["poff"][i]):int(got["poff"][i + 1])].tobytes())
    # bounded calls on every route
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    bounds = [[6, 12], [3], [], [9], []]
    ref = run(make(d, lattice=True), "whole", sents, bounds)
    check_exact(bo, sents, ref, 1.0, [tuple(b) for b in bounds])
    for route in ("chunked", "device"):
        got = run(make(d, route, chunk=2), route, sents, bounds)
        for k in ("poff", "ptok", "pprob", "pgain"):
            assert got[k].tobytes() == ref[k].tobytes(), (route, k)


def same(a, b, keys=("poff", "ptok", "pprob", "pgain")):
    for k in keys:
        assert a[k].tobytes() == b[k].tobytes(), k


def test_routes_byte_for_byte(golden):
    """Every route, chunk size, layout and Viterbi kernel, and the lattice, sampling or uncertainty on: the same
    bytes as the whole-batch call."""
    d, od, r = golden_dicts(golden, True)
    sents = golden_sents(golden) * 20 + [""] * 70 + ["東京 都  " * 9] * 5 + golden_sents(golden) * 10
    ref = run(make(d), "whole", sents)
    for route in ("chunked", "device", "compact", "small", "viterbi0", "unpruned"):
        same(ref, run(make(d, route), route, sents))
    for chunk in (16, 100, 1000):
        same(ref, run(make(d, "chunked", chunk=chunk), "chunked", sents))
    for lanes in (4, 16, 32):
        for sort in (0, 1, 2):
            for kernel in ("whole", "viterbi0", "unpruned"):
                same(ref, run(make(d, kernel, lanes=lanes, sort=sort), kernel, sents))
    for kw in (dict(lattice=True), dict(samples=3), dict(unc=2), dict(lattice=True, samples=2, unc=1)):
        for route in ("whole", "chunked", "device"):
            same(ref, run(make(d, route, **kw), route, sents))


@pytest.mark.parametrize("route", ["multi", "multi_device"])
def test_multi_device(golden, route):
    d, od, r = golden_dicts(golden, True)
    sents = golden_sents(golden) * 40 + [""] * 70 + golden_sents(golden) * 30
    ref = run(make(d), "whole", sents)
    same(ref, run(make(d, route), "device" if route == "multi_device" else "whole", sents))


@pytest.mark.parametrize("gamma", [0.0, 1.0, 8.0])
def test_other_outputs_unchanged(golden, gamma):
    """Tokens, marginals, lattice, samples, uncertainty and text are byte-identical with posterior decoding on and off."""
    d, od, r = golden_dicts(golden, True)
    sents = golden_sents(golden) * 3
    utf8, off = adv.pack(sents)
    outs = []
    for on in (False, True):
        tok = vb.Tokenizer.new(d).marginals(THETA).sampling(2, THETA, seed=9).output_mode("mecab")
        tok.lattice(True).uncertainty(True, boundary_probs=True)
        if on:
            tok.posterior(gamma)
        res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
        outs.append([res.tokens.tobytes(), res.token_probs.tobytes(), res.path_probs.tobytes(), res.samples.tobytes(),
                     res.nodes.tobytes(), res.node_links.tobytes(), res.node_probs.tobytes(), res.entropies.tobytes(),
                     res.boundary_probs.tobytes(), res.text()[1]])
        assert (res.posterior_tokens is None) != on
    assert outs[0] == outs[1]
    for on in (False, True):  # without the rest, and where the eager small-batch path would run
        tok = vb.Tokenizer.new(d).marginals(THETA)
        if on:
            tok.posterior(gamma)
        res = tok.tokenize_batch(["京都東京都京都", "", "に"])
        outs.append((res.tokens.tobytes(), res.token_probs.tobytes(), res.path_probs.tobytes()))
    assert outs[-1] == outs[-2]


def _micro(p):
    m = np.clip(np.rint(np.asarray(p, dtype=np.float64) * 1e6), 0, 1e6).astype(np.int64)
    return [f"{x // 1000000}.{x % 1000000:06d}".encode() for x in m]


@pytest.mark.parametrize("mode", ["mecab", "wakati", "detail", "format"])
def test_posterior_text(golden, mode):
    """The text renders the posterior records as format_oracle renders them; %pP prints the posterior marginal."""
    import format_oracle as fo
    d, od, r = golden_dicts(golden, True)
    sents = golden_sents(golden) * 2 + ["東京 都  "]
    utf8, off = adv.pack(sents)
    for route in ("whole", "chunked"):
        tok = make(d, route, gamma=4.0, text=True, chunk=3)
        if mode == "format":
            tok.output_format("%m\t%pP\t%pc\n")
        else:
            tok.output_mode(mode)
        res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
        t_off, text = res.text()
        if mode == "format":
            exp = fo.format_batch(od, fo.Format("%m\t%pc\n"), utf8, off, res.posterior_offsets, res.posterior_tokens)
            lines = [ln.split(b"\t") for ln in text.split(b"\n")]
            assert [ln[:1] + ln[2:] if len(ln) == 3 else ln for ln in lines] == [ln.split(b"\t") for ln in exp[1].split(b"\n")]
            assert [ln[1] for ln in lines if len(ln) == 3] == _micro(res.posterior_probs)
        else:
            exp = vo.format_batch(od, utf8, off, res.posterior_offsets, res.posterior_tokens, mode)
            assert text == exp[1] and np.array_equal(t_off, exp[0])


def test_posterior_text_refusals(golden):
    d, od, r = golden_dicts(golden, True)
    tok = vb.Tokenizer.new(d).marginals(THETA)
    with pytest.raises(vb.VibratoError, match="needs posterior decoding"):
        tok.set_option("posterior_text", 1)
    tok.posterior(1.0, text=True)
    with pytest.raises(vb.VibratoError, match="posterior text"):
        tok.lattice(True, text=True)
    with pytest.raises(vb.VibratoError, match="posterior text"):
        tok.sampling(2, THETA, text=True)
    with pytest.raises(vb.VibratoError, match="posterior_text"):
        tok.set_option("posterior_text", 2)
    with pytest.raises(vb.VibratoError, match="%pb"):
        tok.output_format("%pb%m\n")
    with pytest.raises(vb.VibratoError, match="posterior_text"):  # the engine refuses it while the text is on
        vb_check(vb_lib().vbt_tokenizer_set_posterior(tok.handle(), 0, 0.0))
    tok.posterior(1.0)  # text off
    tok.lattice(True, text=True)
    with pytest.raises(vb.VibratoError, match="lattice text"):
        tok.set_option("posterior_text", 1)
    tok.lattice(False)
    tok.sampling(2, THETA, text=True)
    with pytest.raises(vb.VibratoError, match="sample text"):
        tok.set_option("posterior_text", 1)


def test_edge_cases():
    """Empty sentences (also in runs across chunk edges), an empty batch, and a sentence of T(900) equally likely
    paths, whose path_prob underflows to 0 while its marginals stay finite."""
    z = adv.zero_dictionary()
    dev = vb.SystemDictionaryBuilder.from_readers(z.lex_csv, z.matrix, z.char_def, z.unk_def)
    bo = BoundedOracle(vo.OracleDictionary(z.lex_csv, z.matrix, z.char_def, z.unk_def), z.char_def, z.unk_def)
    sents = ["", "a" * 900, "b", "", "aab"]
    tok = make(dev, gamma=2.0, lattice=True)
    got = run(tok, "whole", sents)
    assert check_exact(bo, sents, got, 2.0) == 3
    assert got["pgain"][0] == 0.0 and got["pgain"][3] == 0.0
    assert tok.tokenize_batch(sents).path_probs[1] == 0.0
    sents = [""] * 7 + sents + [""] * 5
    got = run(make(dev, gamma=2.0), "whole", sents)
    for route in ("chunked", "device"):
        same(got, run(make(dev, route, gamma=2.0, chunk=2), route, sents))
    for route in ("whole", "device"):
        g = run(make(dev), route, [])
        assert g["poff"].tolist() == [0] and len(g["ptok"]) == 0 and len(g["pgain"]) == 0


def test_no_path(golden):
    d, od, r = golden_dicts(golden, True)
    got = run(make(d), "whole", ["ぬぬ京都", "京都"], spans=[[(0, 6, None)], []])
    assert got["pgain"][0] == -math.inf and int(got["poff"][1]) == 0 and int(got["poff"][2]) > 0


def test_errors_replay_and_accessors(golden):
    d, od, r = golden_dicts(golden, True)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    tok = vb.Tokenizer.new(d)
    with pytest.raises(vb.VibratoError, match="needs marginals"):
        tok.posterior(1.0)
    tok.marginals(THETA)
    for bad in (-1.0, math.inf, math.nan):
        with pytest.raises(vb.VibratoError, match="gamma"):
            tok.posterior(bad)
    tok.posterior(3.0)
    with pytest.raises(vb.VibratoError, match="posterior decoding needs marginals"):
        tok.marginals(0)
    sents = ["京都東京都京都", "", "東京に行った。"]
    res = tok.tokenize_batch(sents)
    tok.ignore_space(True).ignore_space(False)  # rebuilds the engine: the setting is replayed
    res2 = tok.tokenize_batch(sents)
    for k in ("posterior_offsets", "posterior_tokens", "posterior_probs", "posterior_gains"):
        assert getattr(res, k).tobytes() == getattr(res2, k).tobytes(), k
    toks = res.sentence_posterior(0)
    assert [t.prob() for t in toks] == [float(x) for x in res.posterior_probs[:len(toks)]]
    assert "".join(t.surface() for t in toks) == sents[0] and res.sentence_posterior(1) == []
    w = tok.new_worker()
    w.reset_sentence(sents[0])
    w.tokenize()
    assert w.num_posterior_tokens() == len(toks)
    assert [w.posterior_token(k).surface() for k in range(len(toks))] == [t.surface() for t in toks]
    assert w.posterior_token(0).prob() == toks[0].prob()
    tok.posterior(None)
    tok.marginals(0)  # allowed again
    assert tok.tokenize_batch(sents).posterior_tokens is None
    with pytest.raises(vb.VibratoError, match="no posterior"):
        w.num_posterior_tokens()
    import torch
    x = torch.from_numpy(np.frombuffer("京都".encode(), np.uint8).copy()).cuda()
    o = torch.tensor([0, 6], dtype=torch.int64).cuda()
    plain = vb.Tokenizer.new(d).marginals(THETA)
    plain.tokenize_batch_device(x.data_ptr(), o.data_ptr(), 1, 6)
    with pytest.raises(vb.VibratoError, match="posterior"):
        plain.last_device_posterior()
    plain.posterior(1.0)
    plain.tokenize_batch_device(x.data_ptr(), o.data_ptr(), 1, 6)
    do, dt, dp, dg, n = plain.last_device_posterior()
    recs, probs, v = po.sentence_posterior(bo, "京都".encode(), 1.0, theta=THETA)
    assert n == len(recs) and d2h(dt, n, vb.TOKEN_DTYPE).tobytes() == recs.tobytes()



def test_tokenize_cli_posterior(golden, tmp_path):
    """`tokenize -m -t F --posterior G` prints the posterior text of the Python API on every batch size, device list,
    -F, -p and --boundary-marker."""
    import os
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vibrato_b200", "bin", "tokenize")
    for k, v in golden["resources"].items():
        (tmp_path / k).write_text(v, encoding="utf-8", newline="")
    d, od, _ = golden_dicts(golden, True)
    lines = ["京都東京都京都", "東京 都", "", "kampersanda", "東京県に行く", "", "京都 東京"] * 3
    text = ("\n".join(lines) + "\n").encode()
    base = [exe, "-i", str(tmp_path), "-u", str(tmp_path / "user.csv"), "-m", "-t", "0.001", "--posterior", "4"]
    flag_sets = [["--batch-lines", "1"], ["--batch-lines", "7"], ["--batch-lines", "65536"], ["--devices", "0"]]
    flag_sets.append(["--devices", shard_devices_arg(2)])
    for flags, style in ((["-O", "wakati"], "wakati"), (["-O", "detail"], "detail"), (["-F", "%m\t%pP\t%pc\n"], None)):
        tok = vb.Tokenizer.new(d).marginals(0.001).posterior(4.0, text=True)
        if style:
            tok.output_mode(style)
        else:
            tok.output_format("%m\t%pP\t%pc\n")
        expected = tok.tokenize_batch(lines).text()[1]
        for extra in flag_sets:
            p = subprocess.run(base + flags + extra, input=text, capture_output=True, timeout=120)
            assert p.returncode == 0, p.stderr.decode()
            assert p.stdout == expected, (flags, extra)
    marked = ["京都|東京都京都", "東京 都", "", "東京|県に行く"]
    sents = [s.replace("|", "") for s in marked]
    bounds = [[s.encode().index(b"|")] if "|" in s else [] for s in marked]
    tok = vb.Tokenizer.new(d).marginals(0.001).posterior(4.0, text=True).output_mode("wakati")
    expected = tok.tokenize_batch(sents, boundaries=bounds).text()[1]
    p = subprocess.run(base + ["-O", "wakati", "--boundary-marker", "|"], input=("\n".join(marked) + "\n").encode(),
                       capture_output=True, timeout=120)
    assert p.returncode == 0 and p.stdout == expected, p.stderr.decode()
    p = subprocess.run(base + ["-O", "wakati", "-p"], input="京都東京都京都\nEOS\n京都\t*\n東京都京都\nEOS\n".encode(),
                       capture_output=True, timeout=120)
    assert p.returncode == 0, p.stderr.decode()
    spans = [[], [(0, 6, None)]]
    exp = tok.tokenize_batch(["京都東京都京都", "京都東京都京都"], spans=spans).text()[1]
    assert p.stdout == exp


def test_evaluate_cli_posterior(golden, tmp_path):
    """`evaluate --theta F --posterior G` scores the posterior tokens: its precision and recall equal the counts of
    the Python API's posterior paths against the corpus."""
    import os
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vibrato_b200", "bin", "evaluate")
    for k, v in golden["resources"].items():
        (tmp_path / k).write_text(v, encoding="utf-8", newline="")
    d, od, _ = golden_dicts(golden, True)
    sents = [s for s in golden_sents(golden) if s.strip()] * 2
    ref_tok = vb.Tokenizer.new(d)
    corpus, refs = [], []
    for s in sents:  # the reference: the best path, with every other token's feature replaced
        toks = ref_tok.tokenize_batch([s]).sentence_tokens(0)
        keys = set()
        for k, t in enumerate(toks):
            feat = t.feature() if k % 2 == 0 else "X,Y"
            corpus.append(f"{t.surface()}\t{feat}")
            keys.add((t.range_char().start, t.range_char().stop, feat))
        corpus.append("EOS")
        refs.append(keys)
    (tmp_path / "corpus.txt").write_text("\n".join(corpus) + "\n", encoding="utf-8")
    for theta, gamma in ((0.001, 8.0), (0.01, 0.0)):
        res = vb.Tokenizer.new(d).marginals(theta).posterior(gamma).tokenize_batch(sents)
        n_ref = n_sys = n_cor = 0
        for i, keys in enumerate(refs):
            sys = {(t.range_char().start, t.range_char().stop, t.feature()) for t in res.sentence_posterior(i)}
            n_ref, n_sys, n_cor = n_ref + len(keys), n_sys + len(sys), n_cor + len(keys & sys)
        p = subprocess.run([exe, "-i", str(tmp_path), "-u", str(tmp_path / "user.csv"), "-t", str(tmp_path / "corpus.txt"),
                            "--theta", str(theta), "--posterior", str(gamma)], capture_output=True, timeout=120)
        assert p.returncode == 0, p.stderr.decode()
        out = dict(ln.split(" = ") for ln in p.stdout.decode().splitlines())
        assert float(out["Precision"]) == n_cor / n_sys and float(out["Recall"]) == n_cor / n_ref, (out, n_cor, n_sys)
