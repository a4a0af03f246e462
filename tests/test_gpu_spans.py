"""Required tokens on the GPU (vbt_tokenize_batch_spans / vbt_tokenize_batch_device_spans): tokens bit-identical to
the span oracle (tests/span_oracle.py) on every route, the guarantee, the invariants against unconstrained and bounded
calls, marginals / lattice / samples over the span lattice, and the input errors."""
import numpy as np
import pytest

import adversarial as adv
import lattice_oracle as lo
import marginal_oracle as mo
import vibrato_b200 as vb
from span_oracle import Constraints, SpanOracle, constraints, csv_fields
from oracle import vibrato_oracle as vo
from test_gpu_bounded import CHUNK_COPIES, d2h, golden_dicts, lead_bytes, make_tokenizer
from test_gpu_sampling import check_parity

pytestmark = pytest.mark.gpu
ROUTES = ("whole", "chunked", "small", "device", "multi", "multi_device")


def span_patterns(so, text, a, b):
    """Patterns worth trying on the characters [a, b) of text: the full features and first fields of the lexicon
    words of exactly that surface, those of the unk.def entries of its first character, and one that matches nothing."""
    out = [None, "名詞,固有名詞", "NOPE,*,*", ""]
    for lt in ((1, 0) if so.has_user else (0,)):
        for wid, end in so.od.common_prefix(text[a:b], lt):
            if end == b - a:
                f = so.feature((lt << 30) | wid)
                out += [f, csv_fields(f.encode())[0][0].decode() + ",*"]
    base = (so.od.char_info(ord(text[a])) >> 18) & 0xFF
    for w in range(so.unk_off[base], so.unk_off[base + 1]):
        out.append(so.feature((2 << 30) | w))
    return out


def make_spans(so, sents, seed, with_bounds=True):
    """Per sentence: random valid spans (some with patterns, some adjacent, some at 0 / len, every 5th sentence one
    span over everything, every 4th none) and explicit boundaries outside them."""
    rng = np.random.default_rng(seed)
    spans, bounds = [], []
    for i, s in enumerate(sents):
        b = s.encode()
        lb = lead_bytes(b)
        c_of = {x: k for k, x in enumerate(lb)}
        ok = [x for x in lb[:-1] if not (so.space_mask and so.od.char_info(ord(s[c_of[x]])) & so.space_mask)]
        sp = []
        if i % 4 == 3 or not ok:
            pass
        elif i % 5 == 4 and ok[0] == 0:
            sp = [(0, len(b))]
        else:
            pts = sorted(set(int(x) for x in rng.choice(lb, size=min(len(lb), int(rng.integers(2, 7))))))
            j = 0
            while j + 1 < len(pts):
                a, e = pts[j], pts[j + 1]
                if a in ok and rng.random() < 0.8:
                    sp.append((a, e))
                    j += 1 if rng.random() < 0.3 else 2  # adjacent spans share the point
                else:
                    j += 1
        recs = []
        for a, e in sp:
            if rng.random() < 0.5:
                pats = span_patterns(so, s, c_of[a], c_of[e])
                recs.append((a, e, pats[int(rng.integers(len(pats)))]))
            else:
                recs.append((a, e))
        inside = {x for a, e, *_ in recs for x in lb if a < x < e}
        free = [x for x in lb if x not in inside]
        bnd = sorted(int(x) for x in rng.choice(free, size=min(2, len(free)))) if with_bounds and i % 3 else []
        if b and not has_path(so, b, Constraints(tuple(bnd), tuple(recs))):
            recs, bnd = [], []  # (unk.def lacks a category: the constrained lattice has no path, which is undefined)
        spans.append(recs)
        bounds.append(bnd)
    return spans, bounds


def has_path(so, sent, cons):
    ends, (row, _), _ = so.lattice(sent, cons)
    return bool(ends[row])


def run(tok, route, sents, spans, bounds):
    utf8, off = adv.pack(sents)
    if route in ("device", "multi_device"):
        import torch
        so_, recs, pats = vb.Tokenizer.pack_spans(spans)
        bo, bnd = vb.Tokenizer.pack_bounds(bounds)
        d_utf8 = torch.from_numpy(utf8.copy()).cuda()
        d_off = torch.from_numpy(off.astype(np.int64)).cuda()
        d_bo = torch.from_numpy(bo.astype(np.int64)).cuda()
        d_bnd = torch.from_numpy(bnd.astype(np.int32)).cuda() if len(bnd) else torch.zeros(1, dtype=torch.int32).cuda()
        d_so = torch.from_numpy(so_.astype(np.int64)).cuda()
        d_sp = (torch.from_numpy(recs.astype(np.int64).astype(np.int32).reshape(-1)).cuda() if len(recs)
                else torch.zeros(3, dtype=torch.int32).cuda())
        torch.cuda.synchronize()
        a, b, n = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), len(sents), len(utf8),
                                            d_bnd_offsets=d_bo.data_ptr(), d_bnd=d_bnd.data_ptr(), n_bnd=len(bnd),
                                            d_span_offsets=d_so.data_ptr(), d_spans=d_sp.data_ptr(),
                                            n_spans=len(recs), patterns=pats)
        return d2h(a, len(sents) + 1, np.uint64), d2h(b, n, vb.TOKEN_DTYPE)
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds, spans=spans)
    if route == "small" and any(spans):  # k_small_batch steps aside for spans
        assert tok.describe()["last_viterbi"] != "k_small_batch"
    return res.tok_offsets.copy(), res.tokens.copy()


def check(tok, route, so, sents, spans, bounds):
    e_off, e_toks = so.tokenize_batch([s.encode() for s in sents], constraints(bounds, spans))
    if route == "chunked":
        k = -(-CHUNK_COPIES // max(1, len(sents)))
        sents, spans, bounds = sents * k, spans * k, bounds * k
        per = np.diff(e_off.astype(np.int64))
        e_off = np.zeros(len(sents) + 1, dtype=np.uint64)
        e_off[1:] = np.cumsum(np.tile(per, k))
        e_toks = np.tile(e_toks, k)
    off, toks = run(tok, route, sents, spans, bounds)
    np.testing.assert_array_equal(off, e_off)
    for name in vb.TOKEN_DTYPE.names:
        np.testing.assert_array_equal(toks[name], e_toks[name], err_msg=name)
    assert_guarantee(sents, spans, off, toks)


def assert_guarantee(sents, spans, off, toks):
    for i, recs in enumerate(spans):
        t = toks[int(off[i]):int(off[i + 1])]
        for a, e, *_ in recs:
            assert sum(1 for x in t if x["start_byte"] == a and x["end_byte"] == e) == 1, (sents[i], a, e)
            assert not any(a < x["start_byte"] < e or a < x["end_byte"] < e for x in t), (sents[i], a, e)


GOLDEN_EXTRA = ["京都東京都京都", "abcdefgh", "東京   都", "東京都 abc 123", "ａｂｃ漢字", "abc 123 xyz"]


@pytest.mark.parametrize("route", ROUTES)
def test_golden_fixture(golden, route):
    sents = [c["input"] for c in golden["tokenizer_cases"]] + GOLDEN_EXTRA
    for user in (False, True):
        d, od, r = golden_dicts(golden, user)
        for isp, mgl in ((False, 0), (True, 0), (False, 2)):
            tok = make_tokenizer(d, route, isp, mgl)
            so = SpanOracle(od, r["char.def"], r["unk.def"], isp, mgl)
            spans, bounds = make_spans(so, sents, 1 + user)
            check(tok, route, so, sents, spans, bounds)
            check(tok, route, so, ["京都東京都京都", "abcdefgh"], [[(0, 6, "名詞,固有名詞"), (6, 15)], [(1, 8)]],
                  [[], [8]])
            check(tok, route, so, sents, [[] for _ in sents], [[] for _ in sents])


@pytest.mark.parametrize("dictionary", list(adv.FAMILIES) + ["raw", "dual"])
def test_adversarial(dictionary):
    if dictionary in adv.FAMILIES:
        ad, connector = adv.make_dictionary(dictionary), "matrix"
    else:
        ad, connector = adv.make_dictionary("wrap", dual=dictionary == "dual"), dictionary
    if connector == "matrix":
        d = vb.SystemDictionaryBuilder.from_readers(ad.lex_csv, ad.matrix, ad.char_def, ad.unk_def)
    else:
        right, left, cost = ad.matrix
        d = vb.SystemDictionaryBuilder.from_readers_with_bigram_info(ad.lex_csv, right, left, cost, ad.char_def,
                                                                     ad.unk_def, dual_connector=connector == "dual")
    od = vo.OracleDictionary(ad.lex_csv, ad.matrix, ad.char_def, ad.unk_def, dual_connector=connector == "dual")
    d.reset_user_lexicon_from_reader(ad.user_csv)
    od.set_user_csv(ad.user_csv)
    sents = adv.make_sentences(ad, 60, seed=5, max_len=80) + [" ", "a  ", "あ ア  ", "", " a"]
    for route in ("whole", "chunked", "device"):
        for isp, mgl in ((False, 0), (True, 2)):
            tok = make_tokenizer(d, route, isp, mgl)
            so = SpanOracle(od, ad.char_def, ad.unk_def, isp, mgl)
            spans, bounds = make_spans(so, sents, 5)
            check(tok, route, so, sents, spans, bounds)


@pytest.mark.parametrize("kernel", [0, 1, 2])
@pytest.mark.parametrize("lanes", [4, 8, 16, 32])
def test_viterbi_variants(golden, kernel, lanes):
    d, od, r = golden_dicts(golden, True)
    sents = [c["input"] for c in golden["tokenizer_cases"]] + GOLDEN_EXTRA
    so = SpanOracle(od, r["char.def"], r["unk.def"])
    spans, bounds = make_spans(so, sents, 7)
    for order in (0, 1, 2):
        tok = vb.Tokenizer.new(d)
        tok.set_option("viterbi_kernel", kernel)
        tok.set_option("lanes_per_sentence", lanes)
        tok.set_option("sort_by_length", order)
        check(tok, "whole", so, sents, spans, bounds)


def test_invariants(golden):
    """Empty span lists give the bounded / plain bytes and kernels; spans on every best-path token, each with its own
    feature, give the same byte ranges and cost."""
    d, od, r = golden_dicts(golden, True)
    so = SpanOracle(od, r["char.def"], r["unk.def"])
    sents = [c["input"] for c in golden["tokenizer_cases"]] + GOLDEN_EXTRA
    utf8, off = adv.pack(sents)
    tok = vb.Tokenizer.new(d)
    plain = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
    n_plain = tok.last_launch_count()
    empty = tok.tokenize_batch(utf8=utf8, byte_offsets=off, spans=[[] for _ in sents])
    assert tok.last_launch_count() == n_plain
    assert plain.tokens.tobytes() == empty.tokens.tobytes()
    _, bounds = make_spans(so, sents, 9)
    bnd = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds)
    n_bnd = tok.last_launch_count()
    both = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds, spans=[[] for _ in sents])
    assert tok.last_launch_count() == n_bnd
    assert bnd.tokens.tobytes() == both.tokens.tobytes()
    forced = []
    for i in range(len(sents)):
        t = plain.tokens[int(plain.tok_offsets[i]):int(plain.tok_offsets[i + 1])]
        forced.append([(int(x["start_byte"]), int(x["end_byte"]), so.feature(int(x["word_idx"]))) for x in t])
    al = tok.tokenize_batch(utf8=utf8, byte_offsets=off, spans=forced)
    assert tok.last_launch_count() == n_plain + 1  # k_mark_spans
    for f in ("start_byte", "end_byte", "total_cost"):
        np.testing.assert_array_equal(al.tokens[f], plain.tokens[f])
    w = vb.Worker(tok)
    w.reset_sentence(sents[0], spans=forced[0])
    w.tokenize()
    assert w.num_tokens() == len(forced[0])


def test_downstream(golden):
    """Marginals, lattice and samples over the span lattice; each span's nodes carry probability 1 in total, every
    sample holds each span's token, and the samples equal the sampling restatement's byte for byte."""
    d, od, r = golden_dicts(golden, True)
    so = SpanOracle(od, r["char.def"], r["unk.def"])
    sents = [c["input"] for c in golden["tokenizer_cases"]] + GOLDEN_EXTRA
    sents = [s for s in sents if s]
    spans, bounds = make_spans(so, sents, 11)
    cons = constraints(bounds, spans)
    enc = [s.encode() for s in sents]
    theta = 1.0 / 700
    tok = vb.Tokenizer.new(d)
    tok.marginals(theta).lattice(True).sampling(4, theta, seed=5)
    res = tok.tokenize_batch(sents, boundaries=bounds, spans=spans)
    e_tp, e_pp = mo.batch_marginals(so, enc, theta, cons)
    mo.assert_f32_close(res.token_probs, e_tp, what="token_probs")
    mo.assert_f32_close(res.path_probs, e_pp, what="path_probs")
    e_off, e_nodes, e_links, e_probs = lo.batch_lattice(so, enc, cons, theta)
    np.testing.assert_array_equal(res.node_offsets, e_off)
    for name in vb.TOKEN_DTYPE.names:
        np.testing.assert_array_equal(res.nodes[name], e_nodes[name], err_msg=name)
    np.testing.assert_array_equal(res.node_links["prev"], e_links["prev"])
    mo.assert_f32_close(res.node_probs, e_probs, what="node_probs")
    for i, recs in enumerate(spans):
        nodes = res.nodes[int(res.node_offsets[i]):int(res.node_offsets[i + 1])]
        probs = res.node_probs[int(res.node_offsets[i]):int(res.node_offsets[i + 1])]
        for a, e, *_ in recs:
            sel = (nodes["start_byte"] == a) & (nodes["end_byte"] == e)
            assert abs(float(probs[sel].astype(np.float64).sum()) - 1.0) < 1e-5, (sents[i], a, e)
        for j in range(4):
            k = i * 4 + j
            smp = res.samples[int(res.sample_offsets[k]):int(res.sample_offsets[k + 1])]
            for a, e, *_ in recs:
                assert sum(1 for x in smp if x["start_byte"] == a and x["end_byte"] == e) == 1
    check_parity(so, sents, (res.sample_offsets, res.samples), 4, theta, 5, bounds=cons)


def test_output_and_counts(golden):
    """Output text, compact records and connid counting on a span call."""
    d, od, r = golden_dicts(golden, False)
    so = SpanOracle(od, r["char.def"], r["unk.def"])
    sents = [c["input"] for c in golden["tokenizer_cases"]] + GOLDEN_EXTRA
    spans, bounds = make_spans(so, sents, 13)
    cons = constraints(bounds, spans)
    e_off, e_toks = so.tokenize_batch([s.encode() for s in sents], cons)
    utf8, off = adv.pack(sents)
    for mode in ("mecab", "wakati", "detail"):
        tok = vb.Tokenizer.new(d).output_mode(mode)
        toff, text = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds, spans=spans).text()
        x_off, x_text = vo.format_batch(od, utf8, off, e_off, e_toks.astype(vb.TOKEN_DTYPE), mode)
        np.testing.assert_array_equal(toff, x_off)
        assert text == x_text, mode
    tok = vb.Tokenizer.new(d)
    tok.output_format("%m\t%f[0]|%pS|%ps-%pe\n", eos="EOS %L\n")
    _, text = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds, spans=spans).text()
    lines, b = [], utf8.tobytes()
    for i in range(len(sents)):
        s0, prev_end = int(off[i]), 0
        for t in e_toks[int(e_off[i]):int(e_off[i + 1])]:
            surf = b[s0 + t["start_byte"]:s0 + t["end_byte"]]
            sp = b[s0 + prev_end:s0 + t["start_byte"]]
            f0 = csv_fields(so.feature(int(t["word_idx"]) if int(t["word_idx"]) >> 30 != 2 else
                                       (2 << 30) | unk_entry(so, t)).encode())[0][0]
            lines.append(surf + b"\t" + f0 + b"|" + sp + b"|" + f"{t['start_byte']}-{t['end_byte']}\n".encode())
            prev_end = int(t["end_byte"])
        lines.append(f"EOS {int(off[i + 1] - off[i])}\n".encode())
    assert bytes(text) == b"".join(lines)
    tok = vb.Tokenizer.new(d)
    tok.set_option("compact_tokens", 1)
    res = tok.tokenize_batch(sents, boundaries=bounds, spans=spans)
    for f in vb.TOKEN_DTYPE.names:
        np.testing.assert_array_equal(res.tokens[f], e_toks[f])
    tok = vb.Tokenizer.new(d)
    tok.init_connid_counter()
    tok.tokenize_batch(sents, boundaries=bounds, spans=spans)
    lid, rid = tok.connid_counts()
    e_lid, e_rid = so.connid_counts([s.encode() for s in sents], cons)
    np.testing.assert_array_equal(lid, e_lid)
    np.testing.assert_array_equal(rid, e_rid)


def unk_entry(so, t):
    """The unk.def entry of an unknown token (its word_idx keeps 16 bits of the entry index)."""
    return [w for w in range(len(so.unk)) if w & 0xFFFF == int(t["word_idx"]) & 0xFFFF][0]


def test_errors(golden):
    d, od, r = golden_dicts(golden, False)
    sents = ["京都東京都京都", "abc def"]
    tok = vb.Tokenizer.new(d)
    bad = [
        [[(3, 3)], []],            # empty
        [[(6, 3)], []],            # reversed
        [[(0, 22)], []],           # past the end
        [[(1, 6)], []],            # off a lead byte
        [[(0, 7)], []],
        [[(0, 9), (6, 12)], []],   # overlapping
        [[(6, 12), (0, 6)], []],   # unsorted
        [[(0, 6, 5)], []],         # no such pattern (packed below)
    ]
    for sp in bad[:-1]:
        with pytest.raises(vb.VibratoError, match="spans"):
            tok.tokenize_batch(sents, spans=sp)
    so_, recs, _ = vb.Tokenizer.pack_spans([[(0, 6)], []])
    recs[0, 2] = 5
    with pytest.raises(vb.VibratoError, match="spans"):
        tok.tokenize_batch(sents, span_offsets=so_, span_records=recs, patterns=["a"])
    with pytest.raises(vb.VibratoError, match="spans"):  # an explicit boundary inside a span
        tok.tokenize_batch(sents, spans=[[(0, 12)], []], boundaries=[[6], []])
    with pytest.raises(vb.VibratoError, match="boundaries"):  # boundary errors come first
        tok.tokenize_batch(sents, spans=[[(3, 3)], []], boundaries=[[1], []])
    with pytest.raises(vb.VibratoError, match="UTF-8"):
        tok.tokenize_batch(utf8=np.frombuffer(b"\xff\xfe", dtype=np.uint8), byte_offsets=[0, 2], spans=[[(3, 3)]])
    tok.ignore_space(True)
    with pytest.raises(vb.VibratoError, match="spans"):  # a span starting at a skipped space
        tok.tokenize_batch(sents, spans=[[], [(3, 7)]])
    with pytest.raises(vb.VibratoError, match="pattern 0, byte 512: field index above 255"):
        tok.tokenize_batch(sents, spans=[[(0, 6, "*," * 256 + "x")], []])
    with pytest.raises(vb.VibratoError, match="more than 16 constrained"):
        tok.tokenize_batch(sents, spans=[[(0, 6, ",".join("x" * 17))], []])
    tok.set_counting(True)
    with pytest.raises(vb.VibratoError, match="counting"):
        tok.tokenize_batch(sents, spans=[[(0, 6)], []])
    tok.set_counting(False)
    so = SpanOracle(od, r["char.def"], r["unk.def"], True)
    check(tok, "whole", so, sents, [[(0, 6)], [(4, 7, "名詞")]], [[], []])



def test_space_skip_into_a_span_is_refused():
    """With ignore_space, a space that shares a second category with the characters after it starts a skip that runs
    through the span's start into the span: the span cannot be honoured and the call fails."""
    char_def = "DEFAULT 0 1 0\nSPACE 0 1 0\nALPHA 1 1 0\n0x0020 SPACE ALPHA\n0x0061..0x007A ALPHA\n"
    unk_def = "DEFAULT,1,1,0,記号\nSPACE,1,1,0,空白\nALPHA,1,1,0,名詞\n"
    d = vb.SystemDictionaryBuilder.from_readers("ab,1,1,100,名詞\n", "2 2\n0 0 0\n0 1 0\n1 0 0\n1 1 0\n", char_def,
                                                unk_def)
    tok = vb.Tokenizer.new(d).ignore_space(True)
    with pytest.raises(vb.VibratoError, match="spans"):  # the skip from ' ' (byte 1) lands on '!' inside [2, 6)
        tok.tokenize_batch(["x abc!"], spans=[[(2, 6)]])
    assert tok.tokenize_batch(["x abc!"], spans=[[(2, 4)]]).n_tokens > 0  # the skip ends at '!', outside [2, 4)


def partial_input(sentences):
    """MeCab partial-analysis lines for sentences given as lists of (text, pattern or None for free text) pieces, and
    the equivalent (text, boundaries, spans) of the API."""
    lines, plain, bnds, spans = [], [], [], []
    for pieces in sentences:
        text, b, sp = b"", [], []
        for piece, pat in pieces:
            start = len(text)
            text += piece.encode()
            b += [start, len(text)]
            if pat is None:
                lines.append(piece)
            else:
                lines.append(piece + "\t" + pat)
                sp.append((start, len(text), None if pat in ("", "*") else pat))
        plain.append(text.decode())
        bnds.append(b)
        spans.append(sp)
    return lines, plain, bnds, spans


def test_tokenize_cli_partial(golden, tmp_path):
    """`tokenize -p`: the same bytes as the API call with the equivalent spans and boundaries, for -O wakati / mecab
    and -F, across --batch-lines and --devices; the usage errors and the empty-token line error."""
    import os
    import subprocess
    from test_gpu_bounded import ROOT, shard_devices_arg
    exe = os.path.join(ROOT, "vibrato_b200", "bin", "tokenize")
    if not os.path.exists(exe):
        pytest.skip("CLIs not built")
    r = golden["resources"]
    for k, v in r.items():
        (tmp_path / k).write_text(v, encoding="utf-8", newline="")
    sents = [[("京都", "名詞,固有名詞"), ("東京都京都", None)], [("東京", "*"), ("都", "")], [("abc", None)],
             [("一橋", None), ("大学大学院", "名詞")], [("東京県", None), ("abc", "*,*")]] * 3
    lines, plain, bnds, spans = partial_input(sents)
    body = []
    for k, pieces in enumerate(sents):
        body += lines[sum(len(p) for p in sents[:k]):sum(len(p) for p in sents[:k + 1])] + ["EOS"]
    text_last = ("\n".join(body[:-1]) + "\n").encode()  # the final sentence without its EOS line
    text = ("\n".join(body) + "\n").encode()
    d, _, _ = golden_dicts(golden, False)
    runs = [["-O", "wakati"], ["-O", "mecab"], ["-F", "%m[%ps]\\n", "--eos-format", "%S\\n"]]
    for opts in runs:
        t = vb.Tokenizer.new(d)
        if opts[0] == "-O":
            t.output_mode(opts[1])
        else:
            t.output_format("%m[%ps]\n", eos="%S\n")
        expect = t.tokenize_batch(plain, boundaries=bnds, spans=spans).text()[1]
        base = [exe, "-i", str(tmp_path), "-p"] + opts
        for extra in [[], ["--batch-lines", "2"], ["--batch-lines", "1"]] + [["--devices", shard_devices_arg(2)]]:
            for inp in (text, text_last):
                out = subprocess.run(base + extra, input=inp, capture_output=True, timeout=120)
                assert out.returncode == 0, out.stderr.decode()
                assert out.stdout == expect, (opts, extra)
    bad = subprocess.run([exe, "-i", str(tmp_path), "-p", "--boundary-marker", "|"], input=text, capture_output=True,
                         timeout=120)
    assert bad.returncode == 2
    empty = subprocess.run([exe, "-i", str(tmp_path), "-p"], input="京都\nEOS\n東京\n\t名詞\nEOS\n".encode(),
                           capture_output=True, timeout=120)
    assert empty.returncode == 1 and b"line 4" in empty.stderr
