"""Near-best lattices on the GPU (option "lattice_margin"): kept nodes, links and margins equal the restatement
(tests/margin_oracle.py) byte for byte on every route, dictionary family, Viterbi kernel, bounded and span call, with
marginals and sampling on and off; tokens, text, marginals and samples do not change with the option; -1 gives the
full lattice; lattice text renders the kept nodes; the CLI and multi-device tokenizers give the same bytes."""
import os
import subprocess

import numpy as np
import pytest

import adversarial as adv
import lattice_oracle as lo
import margin_oracle as mgo
import marginal_oracle as mo
import segment_fixtures as sf
import vibrato_b200 as vb
from bounded_oracle import BoundedOracle
from oracle import vibrato_oracle as vo
from span_oracle import Constraints, SpanOracle
from test_gpu_lattice import ROUTES
from test_gpu_marginals import adversarial_dicts, d2h, golden_dicts, golden_sents, shard_devices, shard_devices_arg

pytestmark = pytest.mark.gpu
THETA = 0.01
BIG = mgo.MAX_MARGIN
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make(d, D, route="whole", isp=False, mgl=0, theta=None, samples=0, text=False):
    tok = vb.Tokenizer.new(d).ignore_space(isp).max_grouping_len(mgl)
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
    if theta:
        tok.marginals(theta)
    if samples:
        tok.sampling(samples, theta or THETA, seed=3)
    return tok.lattice(True, text=text, margin=D)


def run(tok, route, sents, bounds=None, spans=None):
    """(node_off, nodes, links, margins, node_probs or None, tokens, token_probs or None, samples or None)"""
    utf8, off = adv.pack(sents)
    if route == "device":
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
        no, nd, nl, npb, nn = tok.last_device_lattice()
        return (d2h(no, len(sents) + 1, np.uint64), d2h(nd, nn, vb.TOKEN_DTYPE), d2h(nl, nn, vb.LINK_DTYPE),
                d2h(tok.last_device_lattice_margins(), nn, np.int64), d2h(npb, nn, np.float32) if npb else None,
                d2h(b, n, vb.TOKEN_DTYPE), d2h(tok.last_device_marginals()[0], n, np.float32) if npb else None, None)
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds, spans=spans)
    if route == "small":
        assert tok.describe()["last_viterbi"] != "k_small_batch"
    res.close()
    return (res.node_offsets, res.nodes, res.node_links, res.node_margins, res.node_probs, res.tokens, res.token_probs,
            res.samples)


def check(bo, sents, got, D, bounds=None, theta=None, exp=None):
    """exp: the restatement's batch_pruned_lattice, when the caller has it already."""
    exp = exp or mgo.batch_pruned_lattice(bo, [s.encode() for s in sents], D, bounds, theta)
    e_off, e_nodes, e_links, e_margins, e_probs = exp
    off, nodes, links, margins, probs, toks, tp, _ = got
    np.testing.assert_array_equal(off, e_off)
    assert nodes.tobytes() == e_nodes.tobytes()
    assert links.tobytes() == e_links.tobytes()
    assert margins.tobytes() == e_margins.tobytes()
    best = (links["flags"] & vb.NODE_BEST) != 0
    if toks.dtype == vb.TOKEN_DTYPE:
        assert nodes[best].tobytes() == toks.tobytes()  # the guarantee
    if theta:
        mo.assert_f32_close(probs, e_probs, what="node_probs")
        assert probs[best].tobytes() == tp.tobytes()
    else:
        assert probs is None
    return margins


def positive_margins(bo, sents):
    """Two D values from the percentiles of the positive margins of the full lattices."""
    pos = np.concatenate([np.array([m for m in mgo.margins(mo.Lattice(bo, s.encode()))[0].values() if m > 0] or [1])
                          for s in sents if s])
    return sorted({int(np.percentile(pos, 10)), int(np.percentile(pos, 50))})


@pytest.mark.parametrize("route", ROUTES)
def test_routes(golden, route):
    d, od, r = golden_dicts(golden, True)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    sents = golden_sents(golden) * 20 + [""] * 70 + golden_sents(golden) * 10
    for D in [0] + positive_margins(bo, golden_sents(golden)):
        for theta in (None, THETA):
            check(bo, sents, run(make(d, D, route, theta=theta), route, sents), D, theta=theta)


def test_golden_options(golden):
    sents = golden_sents(golden) + ["東京 都  ", "   "]
    for user in (False, True):
        d, od, r = golden_dicts(golden, user)
        for isp, mgl in ((False, 0), (True, 0), (False, 3)):
            bo = BoundedOracle(od, r["char.def"], r["unk.def"], isp, mgl)
            for D in (0, 3000, BIG):
                for theta in (None, THETA):
                    check(bo, sents, run(make(d, D, isp=isp, mgl=mgl, theta=theta), "whole", sents), D, theta=theta)


@pytest.mark.parametrize("family", list(adv.FAMILIES) + ["raw", "dual"])
def test_adversarial(family):
    """The matrix families and the "wrap" dictionaries (Raw and Dual connectors), whose costs run near +-2^31."""
    d, dev, od = adversarial_dicts(family)
    sents = adv.make_sentences(d, 40, seed=7, max_len=40) + [""]
    for isp in (False, True):
        bo = BoundedOracle(od, d.char_def, d.unk_def, isp)
        theta = THETA if family in adv.FAMILIES else 1e-7
        for D in [0, BIG] + positive_margins(bo, sents[:10]):
            check(bo, sents, run(make(dev, D, isp=isp, theta=theta), "whole", sents), D, theta=theta)


@pytest.mark.parametrize("w,c", [(-32768, -32768), (32767, 32767)])
def test_wrapping_path_costs(w, c):
    """Single-path and `aa` sentences whose i32 costs wrap: the best path is kept with the margins the oracle gives
    (some > 0 where the wrapped comparison left the exact minimum), on every Viterbi kernel."""
    sents = ["a" * 33000, "a" * 7, "", " " + "a" * 20000 + "  "]
    for aa in (None, 0):
        files = adv.single_word_dictionary(w, c, with_aa=aa)
        dev = vb.SystemDictionaryBuilder.from_readers(*files)
        for isp in (False, True):
            bo = BoundedOracle(vo.OracleDictionary(*files), files[2], files[3], isp)
            for D in (0, BIG):
                exp = mgo.batch_pruned_lattice(bo, [s.encode() for s in sents], D)
                for route in ("whole", "viterbi0", "unpruned"):
                    got = run(make(dev, D, route, isp=isp), route, sents)
                    margins = check(bo, sents, got, D, exp=exp)
                    if (w, aa, D) == (-32768, 0, 0):
                        assert margins[(got[2]["flags"] & vb.NODE_BEST) != 0].max() > 0


def test_big_rows():
    """Rows of 2^16 entries and more (test_gpu_segments.py's crowded positions and big sources): kept indices past
    u16, and links through the truncated predecessor index."""
    lex, matrix, char_def, unk_def, user, _ = sf.make_dictionary()
    dev = vb.SystemDictionaryBuilder.from_readers(lex, matrix, char_def, unk_def).reset_user_lexicon_from_reader(user)
    od = vo.OracleDictionary(lex, matrix, char_def, unk_def).set_user_csv(user)
    bo = BoundedOracle(od, char_def, unk_def)
    sents = sf.crowd_sentences() + sf.big_sentences()
    for D in (0, BIG):
        exp = mgo.batch_pruned_lattice(bo, [s.encode() for s in sents], D)
        for route in ("whole", "unpruned"):
            check(bo, sents, run(make(dev, D, route), route, sents), D, exp=exp)


def test_bounds_and_spans(golden):
    d, od, r = golden_dicts(golden, True)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    sents = ["京都東京都京都", "abcdefgh", "", "東京に行った。"]
    bounds = [[6, 12], [3], [], [9]]
    for D in (0, 2000, BIG):
        for route in ("whole", "chunked", "device"):
            check(bo, sents, run(make(d, D, route, theta=THETA), route, sents, bounds), D, bounds, THETA)
    so = SpanOracle(od, r["char.def"], r["unk.def"])
    spans = [[(6, 15, None)], [(0, 3, None)], [], [(0, 6, "名詞")]]
    cons = [Constraints((), tuple(s)) for s in spans]
    for D in (0, 2000, BIG):
        check(so, sents, run(make(d, D, theta=THETA), "whole", sents, spans=spans), D, cons, THETA)


def test_marginals_and_sampling_share_the_forward_pass(golden):
    """With sampling (and marginals) on, the margins come from the forward pass they already run."""
    d, od, r = golden_dicts(golden, True)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    sents = golden_sents(golden) * 3
    for theta in (None, THETA):
        check(bo, sents, run(make(d, 1500, theta=theta, samples=2), "whole", sents), 1500, theta=theta)


def test_other_outputs_unchanged(golden):
    """Tokens, text, marginals and samples are byte-identical with the option on and off; -1 is today's lattice."""
    d, od, r = golden_dicts(golden, True)
    sents = golden_sents(golden) * 3
    utf8, off = adv.pack(sents)
    outs = []
    for D in (None, 0, BIG):
        tok = vb.Tokenizer.new(d).marginals(THETA).sampling(2, THETA, seed=9).output_mode("mecab")
        tok.lattice(True, margin=D)
        res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
        outs.append((res.tokens.tobytes(), res.token_probs.tobytes(), res.path_probs.tobytes(), res.samples.tobytes(),
                     res.text()[1]))
        if D is None:
            assert res.node_margins is None
            full = (res.node_offsets.copy(), res.nodes.tobytes(), res.node_links.tobytes(), res.node_probs.tobytes())
    assert outs[0] == outs[1] == outs[2]
    tok = vb.Tokenizer.new(d).marginals(THETA).lattice(True)
    tok.set_option("lattice_margin", 5)
    tok.set_option("lattice_margin", -1)
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
    assert np.array_equal(res.node_offsets, full[0]) and res.nodes.tobytes() == full[1]
    assert res.node_links.tobytes() == full[2] and res.node_probs.tobytes() == full[3]
    # with the lattice off the option changes nothing
    plain = vb.Tokenizer.new(d).tokenize_batch(utf8=utf8, byte_offsets=off)
    tok = vb.Tokenizer.new(d)
    tok.set_option("lattice_margin", 0)
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
    assert res.tokens.tobytes() == plain.tokens.tobytes() and res.nodes is None


@pytest.mark.parametrize("mode", ["wakati", "mecab", "pb"])
def test_lattice_text(golden, mode):
    import format_oracle as fo
    d, od, r = golden_dicts(golden, True)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    sents = golden_sents(golden)
    utf8, off = adv.pack(sents)
    D = 2000
    e_off, e_nodes, e_links, _, _ = mgo.batch_pruned_lattice(bo, [s.encode() for s in sents], D)
    tok = make(d, D, text=True)
    if mode == "pb":
        fmt = "%pb%m\t%pc\n"
        tok.output_format(fmt, bos="BOS\n")
        _, text = tok.tokenize_batch(utf8=utf8, byte_offsets=off).text()
        plain = fo.format_batch(od, fo.Format("%m\t%pc\n", bos="BOS\n"), utf8, off, e_off, e_nodes)[1].split(b"\n")
        stars = iter(b"*" if f & lo.NODE_BEST else b" " for f in e_links["flags"])
        want = b"\n".join(ln if ln in (b"BOS", b"EOS", b"") else next(stars) + ln for ln in plain)
        assert text == want
    else:
        tok.output_mode(mode)
        t_off, text = tok.tokenize_batch(utf8=utf8, byte_offsets=off).text()
        exp = vo.format_batch(od, utf8, off, e_off, e_nodes, mode)
        assert text == exp[1] and np.array_equal(t_off, exp[0])


def test_python_views_and_errors(golden):
    d, od, r = golden_dicts(golden, True)
    tok = make(d, 0, theta=THETA)
    res = tok.tokenize_batch(["京都東京都京都", ""])
    nodes = res.sentence_nodes(0)
    assert [n.margin() for n in nodes] == res.node_margins[:len(nodes)].tolist()
    assert all(n.margin() == 0 for n in nodes)  # D = 0: only minimum-cost paths
    w = tok.new_worker()
    w.reset_sentence("京都東京都京都")
    w.tokenize()
    assert [w.node(i).margin() for i in range(w.num_nodes())] == [n.margin() for n in nodes]
    tok.ignore_space(True)  # rebuilds the engine: the margin is replayed
    assert tok.tokenize_batch(["京都東京都京都"]).node_margins.tolist() == res.node_margins.tolist()
    with pytest.raises(vb.VibratoError, match="lattice_margin must be"):
        tok.set_option("lattice_margin", -2)
    with pytest.raises(vb.VibratoError, match="lattice_margin must be"):
        tok.set_option("lattice_margin", (1 << 62) + 1)
    with pytest.raises(vb.VibratoError):
        tok.lattice(True, margin=-5)
    full = vb.Tokenizer.new(d).lattice(True).tokenize_batch(["京都"])
    assert full.node_margins is None
    with pytest.raises(vb.VibratoError, match="no margins"):
        full.sentence_nodes(0)[0].margin()
    plain = vb.Tokenizer.new(d).lattice(True)
    import torch
    x = torch.from_numpy(np.frombuffer("京都".encode(), np.uint8).copy()).cuda()
    o = torch.tensor([0, 6], dtype=torch.int64).cuda()
    plain.tokenize_batch_device(x.data_ptr(), o.data_ptr(), 1, 6)
    with pytest.raises(vb.VibratoError, match="cost margin"):
        plain.last_device_lattice_margins()


@pytest.mark.parametrize("route", ["multi", "multi_device"])
def test_multi_device(golden, route):
    d, od, r = golden_dicts(golden, True)
    sents = golden_sents(golden) * 40 + [""] * 70 + golden_sents(golden) * 30
    ref = run(make(d, 2000, theta=THETA), "whole", sents)
    tok = vb.Tokenizer.new(d, devices=shard_devices(2)).marginals(THETA).lattice(True, margin=2000)
    got = run(tok, "device" if route == "multi_device" else "whole", sents)
    for a, b in zip(ref, got):
        assert (a is None and b is None) or a.tobytes() == b.tobytes()


def test_cli_cost_margin(golden, tmp_path):
    exe = os.path.join(ROOT, "vibrato_b200", "bin", "tokenize")
    if not os.path.exists(exe):
        pytest.skip("CLIs not built")
    r = golden["resources"]
    for k, v in r.items():
        (tmp_path / k).write_text(v, encoding="utf-8", newline="")
    lines = ["京都東京都京都", "東京 都", "", "kampersanda", "東京|県に行く"] * 3
    data = ("\n".join(lines) + "\n").encode()
    plain = [s.replace("|", "") for s in lines]
    bnds = [[len(s[:s.index("|")].encode())] if "|" in s else [] for s in lines]
    d, _, _ = golden_dicts(golden, True)
    base = [exe, "-i", str(tmp_path), "-u", str(tmp_path / "user.csv")]
    devs = [["--devices", shard_devices_arg(2)]]
    for D in (0, 2000):
        want = make(d, D, text=True).output_mode("wakati").tokenize_batch(plain, boundaries=bnds).text()[1]
        fmt = "%pb%m\t%pP\n"
        want_fmt = make(d, D, theta=THETA, text=True).output_format(fmt).tokenize_batch(plain, boundaries=bnds).text()[1]
        for flags in [[], ["--batch-lines", "4"], ["--batch-lines", "1"]] + devs:
            p = subprocess.run(base + ["-a", "--cost-margin", str(D), "-O", "wakati", "--boundary-marker", "|"] + flags,
                               input=data, capture_output=True, timeout=120)
            assert p.returncode == 0, p.stderr.decode()
            assert p.stdout == want
            p = subprocess.run(base + ["-a", "--cost-margin", str(D), "-m", "-t", str(THETA), "-F", fmt,
                                       "--boundary-marker", "|"] + flags, input=data, capture_output=True, timeout=120)
            assert p.returncode == 0, p.stderr.decode()
            assert p.stdout == want_fmt
