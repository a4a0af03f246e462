"""Segmentation sampling on the GPU (vbt_tokenizer_set_sampling): the samples match the FFBS restatement
(tests/sampling_oracle.py) up to each sample's first ambiguous draw, they are byte-identical on every route, their
frequencies follow P(path), and switching sampling on changes no other output."""
import collections
import ctypes as C
import math

import numpy as np
import pytest
from scipy import stats

import adversarial as adv
import marginal_oracle as mo
import sampling_oracle as so
import vibrato_b200 as vb
from bounded_oracle import BoundedOracle
from test_gpu_marginals import adversarial_dicts, d2h, golden_dicts, golden_sents, shard_devices
from vibrato_b200 import synth
from vibrato_b200._native import lib
from oracle import vibrato_oracle as vo

pytestmark = pytest.mark.gpu
ROUTES = ("whole", "chunked", "compact", "small", "device", "viterbi0", "unpruned", "multi", "multi_device")
THETA = 0.001
SEEDS = (0, 1, 2 ** 64 - 1)
ambiguous = {"samples": 0}  # samples compared only up to an ambiguous draw, over the session


def make_tokenizer(d, route, n, theta=THETA, seed=0, ignore_space=False, mgl=0):
    tok = vb.Tokenizer.new(d, devices=shard_devices(2)) if route.startswith("multi") else vb.Tokenizer.new(d)
    tok.ignore_space(ignore_space).max_grouping_len(mgl)
    if route == "chunked":
        tok.set_option("chunk_sentences", 64)
    if route == "compact":
        tok.compact_tokens(True)
    if route == "small":
        tok.small_batch(65536)
    if route == "viterbi0":
        tok.set_option("viterbi_kernel", 0)
    if route == "unpruned":
        tok.set_option("viterbi_kernel", 2)
    if route == "retry":  # a pool far too small: the batch is re-run with the same draws
        tok.set_option("pool_estimate_permille", 1)
    return tok.sampling(n, theta, seed) if n else tok


def run(tok, route, sents, bounds=None):
    """(sample_offsets, samples) of one call on `route`."""
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
        tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), len(sents), len(utf8), **kw)
        so_ptr, s_ptr, n = tok.last_device_samples()
        return d2h(so_ptr, len(sents) * tok._sampling[0] + 1, np.uint64), d2h(s_ptr, n, vb.TOKEN_DTYPE)
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds)
    if route == "small":
        assert tok.describe()["last_viterbi"] != "k_small_batch"
    res.close()
    return res.sample_offsets, res.samples


KEY = ("start_char", "end_char", "start_byte", "end_byte", "word_idx")


def check_parity(bo, sents, got, n, theta, seed, bounds=None, expected=None):
    """Every sample equals the restatement's byte for byte; after an ambiguous draw t only its last t records (the
    draws before it) are compared, without their prefix costs.  `expected`: the restatement's samples by sentence
    index, when the caller has them already (so.sentence_samples of the same arguments)."""
    off, recs = got
    assert len(off) == len(sents) * n + 1 and int(off[-1]) == len(recs)
    for i, s in enumerate(sents):
        if expected is not None:
            exp = expected[i]
        else:
            exp = so.sentence_samples(bo, s.encode(), n, theta, seed, i, bounds[i] if bounds else ())
        for j, (rec, _, amb) in enumerate(exp):
            g = recs[int(off[i * n + j]):int(off[i * n + j + 1])]
            if amb is None:
                assert g.tobytes() == rec.tobytes(), (s, j, g, rec)
                continue
            ambiguous["samples"] += 1
            if amb:
                for name in KEY:
                    np.testing.assert_array_equal(g[name][len(g) - amb:], rec[name][len(rec) - amb:], err_msg=name)


def golden_oracle(od, r, isp=False, mgl=0):
    return BoundedOracle(od, r["char.def"], r["unk.def"], isp, mgl)


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("seed", SEEDS)
def test_parity_golden(golden, n, seed):
    sents = golden_sents(golden) + ["東京都に行った。", "あ", "京都 東京"]
    for user in (False, True):
        d, od, r = golden_dicts(golden, user)
        for isp, mgl in ((False, 0), (True, 0), (False, 3)):
            tok = make_tokenizer(d, "whole", n, seed=seed, ignore_space=isp, mgl=mgl)
            check_parity(golden_oracle(od, r, isp, mgl), sents, run(tok, "whole", sents), n, THETA, seed)


def test_parity_bounded(golden):
    d, od, r = golden_dicts(golden, False)
    sents = ["京都東京都京都", "アイアイウ", "東京   都", ""] * 5
    bounds = [[12], [6], [], []] * 5
    for route in ("whole", "device"):
        tok = make_tokenizer(d, route, 3, seed=1, ignore_space=True)
        check_parity(golden_oracle(od, r, True), sents, run(tok, route, sents, bounds), 3, THETA, 1, bounds)


@pytest.mark.parametrize("ignore_space", [False, True])
@pytest.mark.parametrize("family", list(adv.FAMILIES) + ["raw", "dual"])
def test_parity_adversarial(family, ignore_space):
    d, dev, od = adversarial_dicts(family)
    sents = adv.make_sentences(d, 30, seed=5, max_len=40) + [" ", "a  ", "あ ア  ", "", " a"]
    theta = 0.05 if family in adv.FAMILIES else 1e-6  # the wrap family's costs are near +-2^31
    bo = BoundedOracle(od, d.char_def, d.unk_def, ignore_space)
    for n, seed in ((1, 2 ** 64 - 1), (3, 0)):
        tok = make_tokenizer(dev, "whole", n, theta=theta, seed=seed, ignore_space=ignore_space)
        check_parity(bo, sents, run(tok, "whole", sents), n, theta, seed)


def test_parity_synth():
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
    tok = make_tokenizer(d, "whole", 3, theta=0.0005, seed=1, ignore_space=True, mgl=24)
    check_parity(bo, sents, run(tok, "whole", sents), 3, 0.0005, 1)


@pytest.mark.parametrize("route", ROUTES + ("retry",))
def test_routes_bit_identical(golden, route):
    d, od, r = golden_dicts(golden, True)
    sents = golden_sents(golden) * 40 + [""] * 70 + golden_sents(golden) * 30  # empty runs across chunk edges
    if route == "retry":  # more candidates than the smallest pool (2^16 + 4096) holds: the batch provably runs twice
        sents = sents * 12
    ref = run(make_tokenizer(d, "whole", 3, seed=2 ** 64 - 1, ignore_space=True), "whole", sents)
    tok = make_tokenizer(d, route, 3, seed=2 ** 64 - 1, ignore_space=True)
    got = run(tok, route, sents)
    if route == "retry":
        assert tok.describe()["last_reruns"]["pool"] >= 1
    np.testing.assert_array_equal(got[0], ref[0])
    assert got[1].tobytes() == ref[1].tobytes()


@pytest.mark.parametrize("route", ("whole", "chunked", "device", "multi"))
def test_other_outputs_unchanged(golden, route):
    """Tokens, marginals, lattice and text are byte-identical with sampling on and off; the marginals' theta is
    shared."""
    d, _, _ = golden_dicts(golden, True)
    sents = golden_sents(golden) * 20
    outs = []
    for n in (0, 4):
        tok = make_tokenizer(d, route, 0).marginals(THETA)
        if route != "multi":
            tok.lattice(True)
        if route != "device":
            tok.output_mode("mecab")
        if n:
            tok.sampling(n, THETA, 5)
        if route == "device":
            import torch
            utf8, off = adv.pack(sents)
            d_utf8, d_off = torch.from_numpy(utf8.copy()).cuda(), torch.from_numpy(off.astype(np.int64)).cuda()
            torch.cuda.synchronize()
            a, b, nt = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), len(sents), len(utf8))
            tp, pp = tok.last_device_marginals()
            lat = tok.last_device_lattice()
            outs.append([d2h(a, len(sents) + 1, np.uint64), d2h(b, nt, vb.TOKEN_DTYPE), d2h(tp, nt, np.float32),
                         d2h(pp, len(sents), np.float32), d2h(lat[1], lat[4], vb.TOKEN_DTYPE)])
            continue
        res = tok.tokenize_batch(sents)
        text = res.text()[1]
        res.close()
        o = [res.tok_offsets, res.tokens, res.token_probs, res.path_probs, text]
        if route != "multi":
            o += [res.node_offsets, res.nodes, res.node_links, res.node_probs]
        outs.append(o)
    for a, b in zip(*outs):
        if isinstance(a, bytes):
            assert a == b
        else:
            assert a.tobytes() == b.tobytes()


def _path_keys(lat, path):
    return tuple((lat.node(n)[1], n[0], lat.node(n)[2]) for n in path)


def _sample_keys(off, recs, k):
    g = recs[int(off[k]):int(off[k + 1])]
    return tuple((int(x["start_char"]), int(x["end_char"]), int(x["word_idx"])) for x in g)


@pytest.mark.parametrize("sent, theta", [("に", 0.0002), ("東京都", 0.002), ("京都東京都京都", 0.001)])
def test_distribution(golden, sent, theta):
    """200 000 draws (the sentence repeated, n = 1) against the exact P(path), chi-square at a fixed seed."""
    d, od, r = golden_dicts(golden, False)
    lat = mo.Lattice(golden_oracle(od, r), sent.encode())
    paths = mo.all_paths(lat)
    cmin = min(c for c, _ in paths)
    weights = [math.exp(-theta * (c - cmin)) for c, _ in paths]
    z = sum(weights)
    index = {_path_keys(lat, p): k for k, (_, p) in enumerate(paths)}
    draws = 200000
    off, recs = run(make_tokenizer(d, "whole", 1, theta=theta, seed=20261016), "whole", [sent] * draws)
    counts = collections.Counter(index[_sample_keys(off, recs, k)] for k in range(draws))
    expected = [draws * w / z for w in weights]
    big = [k for k, e in enumerate(expected) if e >= 5]
    small = [k for k in range(len(paths)) if k not in big]
    obs = [counts[k] for k in big] + ([sum(counts[k] for k in small)] if small else [])
    exp = [expected[k] for k in big] + ([sum(expected[k] for k in small)] if small else [])
    assert len(obs) >= 2
    p = stats.chisquare(obs, exp).pvalue
    print(f"sampling chi-square {sent}: {len(paths)} paths, p = {p:.4f}")
    assert p > 1e-4


def test_large_theta_limit(golden):
    """theta = 100: a unique minimum-cost path is drawn every time, byte for byte the tokens; where minima tie every
    sample is one of the minimum-cost paths."""
    d, od, r = golden_dicts(golden, False)
    sents = [s for s in golden_sents(golden) if s] + ["東京都に行った。", "あ"]
    bo = golden_oracle(od, r)
    tok = make_tokenizer(d, "whole", 8, theta=100.0, seed=3)
    off, recs = run(tok, "whole", sents)
    toks = vb.Tokenizer.new(d).tokenize_batch(sents)
    unique = 0
    for i, s in enumerate(sents):
        lat = mo.Lattice(bo, s.encode())
        if not lat.ends[lat.eos_row]:  # no path: n empty samples (test_edge_cases)
            continue
        r_eos = so.forward(lat, 100.0)[2]
        best = lat.best_path()
        if so.path_cost(lat, best) != r_eos:
            continue
        t = toks.tokens[int(toks.tok_offsets[i]):int(toks.tok_offsets[i + 1])]
        n_min = sum(1 for c, _ in mo.all_paths(lat, limit=10 ** 6) if c == r_eos) if len(s) <= 12 else None
        for j in range(8):
            g = recs[int(off[i * 8 + j]):int(off[i * 8 + j + 1])]
            if n_min == 1:
                assert g.tobytes() == t.tobytes(), s
        unique += n_min == 1
    assert unique
    d2, dev, od2 = adversarial_dicts("ties")
    sents = [s for s in adv.make_sentences(d2, 40, seed=9, max_len=30) if s]
    bo = BoundedOracle(od2, d2.char_def, d2.unk_def)
    off, recs = run(make_tokenizer(dev, "whole", 16, theta=100.0, seed=4), "whole", sents)
    tied = 0
    for i, s in enumerate(sents):
        lat = mo.Lattice(bo, s.encode())
        node_of = {}
        for n in lat.nodes[1:]:
            node_of.setdefault((lat.node(n)[1], n[0], lat.node(n)[2]), []).append(n)
        if any(len(v) > 1 for v in node_of.values()):
            continue  # a record would not name its node
        r_eos = so.forward(lat, 100.0)[2]
        tied += any(0 < f < 1 for f in mo.tie_fractions(lat).values())
        for j in range(16):
            path = [node_of[k][0] for k in _sample_keys(off, recs, i * 16 + j)]
            assert so.path_cost(lat, path) == r_eos, s
    assert tied


def test_edge_cases(golden):
    d, od, r = golden_dicts(golden, False)
    bo = golden_oracle(od, r)
    for route in ("whole", "device"):
        off, recs = run(make_tokenizer(d, route, 3), route, [])
        assert list(off) == [0] and len(recs) == 0
        off, recs = run(make_tokenizer(d, route, 3), route, ["", "", ""])
        assert list(off) == [0] * 10 and len(recs) == 0
    sents = ["あ", "", "京", "a", "東京都"]
    got = run(make_tokenizer(d, "whole", 1024, seed=9), "whole", sents)
    check_parity(bo, sents, got, 1024, THETA, 9)
    assert all(int(got[0][1024 + j + 1] - got[0][1024 + j]) == 0 for j in range(1024))  # the empty sentence


def test_refusals_and_switch_off(golden):
    d, _, _ = golden_dicts(golden, False)
    tok = vb.Tokenizer.new(d)
    for n, theta in ((1025, 1.0), (1, 0.0), (1, -1.0), (1, float("nan")), (1, float("inf"))):
        with pytest.raises(vb.VibratoError) as e:
            tok.sampling(n, theta)
        assert e.value.kind == "InvalidArgument"
    tok.marginals(0.5)
    with pytest.raises(vb.VibratoError) as e:
        tok.sampling(2, 0.25)
    assert "0.5" in str(e.value) and "0.25" in str(e.value)
    tok.sampling(2, 0.5)
    with pytest.raises(vb.VibratoError) as e:
        tok.marginals(0.75)
    assert "0.75" in str(e.value) and "0.5" in str(e.value)
    res = tok.tokenize_batch(["京都"])
    assert res.samples is not None and res.n_samples == 2
    with pytest.raises(vb.VibratoError):
        res.sentence_samples(0)[0][0].prob()
    tok.sampling(0)
    res = tok.tokenize_batch(["京都"])
    assert res.samples is None and res.token_probs is not None
    a, b, n = C.c_void_p(), C.c_void_p(), C.c_uint64()
    assert lib().vbt_result_samples(res._h, C.byref(a), C.byref(b), C.byref(n)) == 1
    with pytest.raises(vb.VibratoError):
        res.sentence_samples(0)
    with pytest.raises(vb.VibratoError):
        tok.last_device_samples()
    tok.sampling(1024, 0.5)
    with pytest.raises(vb.VibratoError) as e:  # n_sent * n >= 2^32
        tok.tokenize_batch([""] * (1 << 22))
    assert e.value.kind == "InvalidArgument"


def test_worker_rebuild_and_launches(golden):
    d, _, _ = golden_dicts(golden, False)
    sents = golden_sents(golden)
    tok = vb.Tokenizer.new(d)
    tok.tokenize_batch(sents)
    n_off, n_stages = tok.last_launch_count(), len(tok.last_stage_ms())
    tok.sampling(3, THETA, 42)
    res = tok.tokenize_batch(sents)
    assert tok.last_launch_count() == n_off + 3 and len(tok.last_stage_ms()) == n_stages
    i = sents.index("京都東京都京都")
    w = tok.new_worker()
    w.reset_sentence("京都東京都京都")
    w.tokenize()
    solo = [[t._r.tobytes() for t in w.sample_tokens(j)] for j in range(3)]
    assert solo[0]  # the worker's sentence is sentence 0 of its own call: its draws are those of index 0
    ref = run(make_tokenizer(d, "whole", 3, seed=42), "whole", ["京都東京都京都"])
    assert b"".join(b"".join(s) for s in solo) == ref[1].tobytes()
    assert [len(x) for x in res.sentence_samples(i)] == [int(res.sample_offsets[i * 3 + j + 1] - res.sample_offsets[i * 3 + j])
                                                         for j in range(3)]
    tok.max_grouping_len(0)  # rebuilds the engine: sampling is replayed
    np.testing.assert_array_equal(tok.tokenize_batch(sents).samples, res.samples)


def test_report_ambiguous():
    """Prints how many samples the tests above compared only up to an ambiguous draw (run in the same session)."""
    print(f"sampling: {ambiguous['samples']} samples with an ambiguous draw")
