"""Lattice output on the GPU (option "lattice"): nodes and links equal the restatement (tests/lattice_oracle.py)
exactly, node marginals match it and equal token_prob bit for bit on the best path, every single-device route gives
the same bytes, the option at 1 leaves tokens, text and marginals as they were, and lattice text renders the nodes."""
import numpy as np
import pytest

import adversarial as adv
import lattice_oracle as lo
import marginal_oracle as mo
import vibrato_b200 as vb
from bounded_oracle import BoundedOracle
from oracle import vibrato_oracle as vo
from test_gpu_marginals import adversarial_dicts, d2h, golden_dicts, golden_sents, shard_devices, shard_devices_arg

pytestmark = pytest.mark.gpu
ROUTES = ("whole", "chunked", "compact", "small", "device", "viterbi0", "unpruned")
THETA = 0.01


def make(d, route="whole", isp=False, mgl=0, theta=None, lattice=1):
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
    if lattice:
        tok.lattice(True, text=lattice == 2)
    return tok


def run(tok, route, sents, bounds=None):
    """(node_off, nodes, links, node_probs or None, tok_off, tokens, token_probs or None)"""
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
        a, b, n = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), len(sents), len(utf8), **kw)
        no, nd, nl, npb, nn = tok.last_device_lattice()
        tp = None
        if npb:
            tp = d2h(tok.last_device_marginals()[0], n, np.float32)
        return (d2h(no, len(sents) + 1, np.uint64), d2h(nd, nn, vb.TOKEN_DTYPE), d2h(nl, nn, vb.LINK_DTYPE),
                d2h(npb, nn, np.float32) if npb else None, d2h(a, len(sents) + 1, np.uint64), d2h(b, n, vb.TOKEN_DTYPE), tp)
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds)
    if route == "small":
        assert tok.describe()["last_viterbi"] != "k_small_batch"
    res.close()
    return (res.node_offsets, res.nodes, res.node_links, res.node_probs, res.tok_offsets, res.tokens, res.token_probs)


def check(bo, sents, got, bounds=None, theta=None):
    e_off, e_nodes, e_links, e_probs = lo.batch_lattice(bo, [s.encode() for s in sents], bounds, theta)
    off, nodes, links, probs, tok_off, toks, tp = got
    np.testing.assert_array_equal(off, e_off)
    assert nodes.tobytes() == e_nodes.tobytes()
    assert links.tobytes() == e_links.tobytes()
    best = (links["flags"] & vb.NODE_BEST) != 0
    if toks.dtype == vb.TOKEN_DTYPE:
        assert nodes[best].tobytes() == toks.tobytes()  # the guarantee
    if theta:
        assert probs is not None and probs.shape == e_probs.shape
        mo.assert_f32_close(probs, e_probs, what="node_probs")
        assert probs[best].tobytes() == tp.tobytes()  # bit for bit
    else:
        assert probs is None


def test_golden_options(golden):
    sents = golden_sents(golden) + ["東京 都  ", "   "]
    for user in (False, True):
        d, od, r = golden_dicts(golden, user)
        for isp, mgl in ((False, 0), (True, 0), (False, 3)):
            bo = BoundedOracle(od, r["char.def"], r["unk.def"], isp, mgl)
            for theta in (None, THETA):
                check(bo, sents, run(make(d, isp=isp, mgl=mgl, theta=theta), "whole", sents), theta=theta)


def test_golden_bounds(golden):
    d, od, r = golden_dicts(golden, True)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    sents = ["京都東京都京都", "abcdefgh", "", "東京に行った。"]
    bounds = [[6, 12], [3], [], [9]]
    for route in ("whole", "chunked", "device"):
        check(bo, sents, run(make(d, route, theta=THETA), route, sents, bounds), bounds, THETA)


@pytest.mark.parametrize("family", list(adv.FAMILIES) + ["raw", "dual"])
def test_adversarial(family):
    d, dev, od = adversarial_dicts(family)
    sents = adv.make_sentences(d, 40, seed=7, max_len=40) + [""]
    for isp in (False, True):
        bo = BoundedOracle(od, d.char_def, d.unk_def, isp)
        theta = THETA if family in adv.FAMILIES else 1e-7
        check(bo, sents, run(make(dev, isp=isp, theta=theta), "whole", sents), theta=theta)


def test_long_sentence(golden):
    """Past 16 000 characters the pruned k_viterbi2 hands over to its unpruned twin."""
    d, od, r = golden_dicts(golden, True)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    sents = ["京都東京都に行った。abc " * 1400, "京都"]
    assert len(sents[0]) > 16000
    check(bo, sents, run(make(d), "whole", sents))


@pytest.mark.parametrize("route", ROUTES)
def test_routes_bit_identical(golden, route):
    d, od, r = golden_dicts(golden, True)
    sents = golden_sents(golden) * 40 + [""] * 70 + golden_sents(golden) * 30
    ref = run(make(d, theta=THETA), "whole", sents)
    got = run(make(d, route, theta=THETA), route, sents)
    for a, b in zip(ref[:4], got[:4]):
        assert a.tobytes() == b.tobytes()
    if route == "whole":
        check(BoundedOracle(od, r["char.def"], r["unk.def"]), sents, got, theta=THETA)


def test_lattice_one_changes_nothing(golden):
    d, od, r = golden_dicts(golden, True)
    sents = golden_sents(golden) * 3
    utf8, off = adv.pack(sents)
    for mode in ("mecab", "detail"):
        outs = []
        for lat in (0, 1):
            tok = make(d, theta=THETA, lattice=lat).output_mode(mode)
            res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
            outs.append((res.tokens.tobytes(), res.token_probs.tobytes(), res.path_probs.tobytes(), res.text()[1]))
        assert outs[0] == outs[1]


@pytest.mark.parametrize("mode", ["mecab", "wakati", "detail", "format"])
def test_lattice_text(golden, mode):
    import format_oracle as fo
    d, od, r = golden_dicts(golden, True)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    sents = golden_sents(golden)
    utf8, off = adv.pack(sents)
    tok = make(d, theta=THETA, lattice=2)
    e_off, e_nodes, _, _ = lo.batch_lattice(bo, [s.encode() for s in sents])
    if mode == "format":  # the oracle has no %pP: its column is checked against the node marginals
        bos = "BOS\n"
        tok.output_format("%m\t%pc\t%pP\t%f[0]\n", bos=bos)
        exp = fo.format_batch(od, fo.Format("%m\t%pc\t%f[0]\n", bos=bos), utf8, off, e_off, e_nodes)
    else:
        tok.output_mode(mode)
        exp = vo.format_batch(od, utf8, off, e_off, e_nodes, mode)
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
    t_off, text = res.text()
    if mode == "format":
        lines = [ln.split(b"\t") for ln in text.split(b"\n")]
        elines = [ln.split(b"\t") for ln in exp[1].split(b"\n")]
        assert [ln[:2] + ln[3:] if len(ln) == 4 else ln for ln in lines] == elines
        pcol = [ln[2] for ln in lines if len(ln) == 4]
        micro = np.clip(np.rint(res.node_probs.astype(np.float64) * 1e6), 0, 1e6).astype(np.int64)
        assert pcol == [f"{m // 1000000}.{m % 1000000:06d}".encode() for m in micro]
    else:
        assert text == exp[1] and np.array_equal(t_off, exp[0])


def test_errors(golden):
    d, od, r = golden_dicts(golden, False)
    tok = vb.Tokenizer.new(d)
    with pytest.raises(vb.VibratoError, match="lattice must be"):
        tok.set_option("lattice", 3)
    tok.output_format("%m%pn\n")
    with pytest.raises(vb.VibratoError, match="change the format before"):
        tok.lattice(True, text=True)
    tok.lattice(True)  # lattice = 1 keeps the text of the tokens: fine
    tok.output_format("%m\n")
    tok.lattice(True, text=True)
    with pytest.raises(vb.VibratoError, match="no previous token"):
        tok.output_format("%pS%m\n")
    res = vb.Tokenizer.new(d).tokenize_batch(["京都"])
    assert res.nodes is None
    with pytest.raises(vb.VibratoError):
        res.sentence_nodes(0)


def test_python_views(golden):
    d, od, r = golden_dicts(golden, False)
    tok = make(d, theta=THETA)
    res = tok.tokenize_batch(["京都東京都京都", ""])
    nodes = res.sentence_nodes(0)
    assert len(nodes) == res.num_nodes(0) and res.num_nodes(1) == 0
    best = [n for n in nodes if n.is_best()]
    toks = res.sentence_tokens(0)
    assert [n.surface() for n in best] == [t.surface() for t in toks]
    assert [n.prob() for n in best] == [t.prob() for t in toks]
    assert nodes[0].prev() is None or nodes[nodes[0].prev()].range_char().stop <= nodes[0].range_char().start
    w = tok.new_worker()
    w.reset_sentence("京都東京都京都")
    w.tokenize()
    assert w.num_nodes() == len(nodes) and [n.surface() for n in w.node_iter()] == [n.surface() for n in nodes]


def test_pb_format(golden):
    """%pb prints '*' on the best path and ' ' elsewhere in lattice text; outside it, it keeps its old error."""
    d, od, r = golden_dicts(golden, True)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    sents = golden_sents(golden)
    tok = make(d, theta=THETA, lattice=2).output_format("%pb%m\t%pP\n", bos="BOS\n")
    res = tok.tokenize_batch(sents)
    _, text = res.text()
    _, e_nodes, e_links, _ = lo.batch_lattice(bo, [s.encode() for s in sents])
    want = bytearray()
    k = 0
    for i, s in enumerate(sents):
        want += b"BOS\n"
        for _ in range(int(res.node_offsets[i + 1] - res.node_offsets[i])):
            nd = e_nodes[k]
            star = b"*" if e_links["flags"][k] & lo.NODE_BEST else b" "
            m = int(np.clip(np.rint(float(res.node_probs[k]) * 1e6), 0, 1e6))
            want += star + s.encode()[nd["start_byte"]:nd["end_byte"]] + f"\t{m // 1000000}.{m % 1000000:06d}\n".encode()
            k += 1
        want += b"EOS\n"
    assert text == bytes(want)
    with pytest.raises(vb.VibratoError, match="change the format before"):
        tok.lattice(True, text=False)
    plain = vb.Tokenizer.new(d)
    with pytest.raises(vb.VibratoError, match="%pb has no value"):
        plain.output_format("%pb%m\n")
    lat2 = vb.Tokenizer.new(d).lattice(True, text=True)
    with pytest.raises(vb.VibratoError, match=r"byte 2: %pn has no value in lattice text"):
        lat2.output_format("%m%pn\n")


@pytest.mark.parametrize("route", ["multi", "multi_device"])
def test_multi_device(golden, route):
    d, od, r = golden_dicts(golden, True)
    sents = golden_sents(golden) * 40 + [""] * 70 + golden_sents(golden) * 30
    ref = run(make(d, theta=THETA), "whole", sents)
    tok = vb.Tokenizer.new(d, devices=shard_devices(2)).marginals(THETA).lattice(True)
    got = run(tok, "device" if route == "multi_device" else "whole", sents)
    for a, b in zip(ref, got):
        assert a.tobytes() == b.tobytes()
    if route == "multi":  # lattice text is merged like the tokens' text
        single = make(d, lattice=2).output_mode("mecab").tokenize_batch(sents).text()[1]
        multi = vb.Tokenizer.new(d, devices=shard_devices(2)).lattice(True, text=True).output_mode("mecab").tokenize_batch(sents)
        assert multi.text()[1] == single


def test_cli_all_morphs(golden, tmp_path):
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "vibrato_b200", "bin", "tokenize")
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
    want_mecab = make(d, lattice=2).output_mode("mecab").tokenize_batch(plain, boundaries=bnds).text()[1]
    fmt = "%pb%m\t%pP\n"
    want_fmt = make(d, theta=THETA, lattice=2).output_format(fmt).tokenize_batch(plain, boundaries=bnds).text()[1]
    devs = [["--devices", shard_devices_arg(2)]]
    for flags in [[], ["--batch-lines", "4"], ["--batch-lines", "1"]] + devs:
        p = subprocess.run(base + ["-a", "-O", "mecab", "--boundary-marker", "|"] + flags, input=data, capture_output=True,
                           timeout=120)
        assert p.returncode == 0, p.stderr.decode()
        assert p.stdout == want_mecab
        p = subprocess.run(base + ["--all-morphs", "-m", "-t", str(THETA), "-F", fmt, "--boundary-marker", "|"] + flags,
                           input=data, capture_output=True, timeout=120)
        assert p.returncode == 0, p.stderr.decode()
        assert p.stdout == want_fmt
