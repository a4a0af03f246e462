"""The front end on the GPU at the edges of char.def and UTF-8 (k_front, k_candidates*, k_candidate_stats,
k_small_batch, k_mark_spans): the families of tests/charclass_fixtures.py — characters in 2-4 categories, SPACE as a
secondary category, pairwise chains, categories 16 and 17, ids that spill into the base id and flag bits, U+0000's
class for astral characters — tokenized byte-identically to the C oracle on every route, with boundaries and spans
against the bounded and span oracles, marginals, lattice and uncertainty against their oracles, and every invalid
UTF-8 shape refused."""
import functools

import numpy as np
import pytest

import charclass_fixtures as cf
import test_gpu_lattice as gl
import test_gpu_uncertainty as gu
import vibrato_b200 as vb
from bounded_oracle import BoundedOracle
from oracle import vibrato_oracle as vo
from span_oracle import Constraints, SpanOracle
from test_gpu_bounded import d2h, lead_bytes
from test_gpu_marginals import shard_devices

pytestmark = pytest.mark.gpu
ROUTES = ("whole", "chunked", "device", "compact", "small", "viterbi0", "unpruned", "multi", "multi_device")
SETTINGS = [(isp, mgl) for isp in (False, True) for mgl in cf.MGLS]
SMALL_BYTES = 16384  # host batches of at most this much text take k_small_batch


@functools.lru_cache(maxsize=None)
def family(name):
    """(fixture, device dictionary, oracle dictionary), user lexicon included."""
    f = cf.make_family(name)
    d = vb.SystemDictionaryBuilder.from_readers(*f.sources())
    d.reset_user_lexicon_from_reader(f.user_csv)
    od = vo.OracleDictionary(*f.sources())
    od.set_user_csv(f.user_csv)
    return f, d, od


def sentences(f, max_chars=None):
    return [s for s in cf.sentences(f).values() if max_chars is None or len(s) <= max_chars]


def assert_same(off, toks, e_off, e_toks, what=""):
    np.testing.assert_array_equal(off, e_off, err_msg=what)
    assert len(toks) == len(e_toks), what
    for name in vb.TOKEN_DTYPE.names:
        np.testing.assert_array_equal(toks[name], e_toks[name], err_msg=f"{what} {name}")


def device_call(tok, sents):
    import torch
    utf8, off = vb.Tokenizer.pack(sents)
    d_utf8 = torch.from_numpy(utf8.copy() if len(utf8) else np.zeros(1, np.uint8)).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    torch.cuda.synchronize()
    a, b, n = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), len(sents), len(utf8))
    return d2h(a, len(sents) + 1, np.uint64), d2h(b, n, vb.TOKEN_DTYPE)


def tokenizer(d, route, isp=False, mgl=0):
    tok = vb.Tokenizer.new(d, devices=shard_devices(2)) if route.startswith("multi") else vb.Tokenizer.new(d)
    tok.ignore_space(isp).max_grouping_len(mgl)
    if route == "chunked":
        tok.set_option("chunk_sentences", 7)
    if route == "compact":
        tok.compact_tokens(True)
    if route == "small":
        tok.small_batch(65536)
    if route == "viterbi0":
        tok.set_option("viterbi_kernel", 0)
    if route == "unpruned":
        tok.set_option("viterbi_kernel", 2)
    return tok


EXPECTED_ROUTE = {"whole": "k_viterbi2", "chunked": "k_viterbi2", "device": "k_viterbi2", "compact": "k_viterbi2",
                  "small": "k_small_batch", "viterbi0": "k_viterbi", "unpruned": "k_viterbi2_unpruned"}


def run_route(tok, route, sents):
    """(tok_off, tokens) of one call; asserts the Viterbi kernel the route claims."""
    if route in ("device", "multi_device"):
        off, toks = device_call(tok, sents)
    else:
        utf8, off = vb.Tokenizer.pack(sents)
        res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
        off, toks = res.tok_offsets.copy(), res.tokens.copy()
    if route in EXPECTED_ROUTE and sents:
        assert tok.describe()["last_viterbi"] == EXPECTED_ROUTE[route], route
    return off, toks


def batches(route, sents):
    """The sentences as one batch, or, for "small", as batches of at most SMALL_BYTES of text."""
    if route != "small":
        return [sents]
    out, cur, size = [], [], 0
    for s in sents:
        n = len(s.encode() if isinstance(s, str) else s)
        if cur and size + n > SMALL_BYTES:
            out.append(cur)
            cur, size = [], 0
        cur.append(s)
        size += n
    return out + [cur]


@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("name", cf.FAMILIES)
def test_tokens_match_oracle(name, route):
    """Every fixture sentence, with and without ignore_space, at every max_grouping_len, byte-identical to the
    oracle."""
    f, d, od = family(name)
    sents = sentences(f)
    for isp, mgl in SETTINGS:
        tok = tokenizer(d, route, isp, mgl)
        for batch in batches(route, sents):
            utf8, off = vb.Tokenizer.pack(batch)
            e_off, e_toks, _ = od.tokenize_batch(utf8, off, isp, mgl)
            got = run_route(tok, route, batch)
            assert_same(*got, e_off, e_toks, f"{name} {route} ignore_space={isp} mgl={mgl}")


@pytest.mark.parametrize("name", cf.FAMILIES)
def test_lanes_and_sort_orders(name):
    """lanes_per_sentence 4 / 8 / 16 / 32 x sort_by_length 0 / 1 / 2, with the space skip on."""
    f, d, od = family(name)
    sents = sentences(f)
    utf8, off = vb.Tokenizer.pack(sents)
    for isp, mgl in ((True, 0), (False, 3)):
        e_off, e_toks, _ = od.tokenize_batch(utf8, off, isp, mgl)
        tok = tokenizer(d, "whole", isp, mgl)
        for lanes in (4, 8, 16, 32):
            for sort in (0, 1, 2):
                tok.set_option("lanes_per_sentence", lanes)
                tok.set_option("sort_by_length", sort)
                assert_same(*run_route(tok, "whole", sents), e_off, e_toks, f"lanes={lanes} sort={sort}")


@pytest.mark.parametrize("name", cf.FAMILIES)
def test_long_sentence_and_large_tile(name):
    """A sentence of more than 16 000 characters (the unpruned twin) and a tile of more than kFrontStage bytes."""
    f, d, od = family(name)
    for sents, route in (([cf.long_sentence(), "ab"], "k_viterbi2_unpruned"), (cf.tile_batch(), "k_viterbi2")):
        utf8, off = vb.Tokenizer.pack(sents)
        for isp, mgl in ((False, 0), (True, 3)):
            e_off, e_toks, _ = od.tokenize_batch(utf8, off, isp, mgl)
            tok = tokenizer(d, "whole", isp, mgl)
            res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
            assert tok.describe()["last_viterbi"] == route
            assert_same(res.tok_offsets, res.tokens, e_off, e_toks, route)


@pytest.mark.parametrize("name", cf.FAMILIES)
def test_counters_and_connid_counts(name):
    """The counted run (k_candidate_stats' copy of the skip and of gen_unknown) against the oracle's counters, and
    connid_counting against BoundedOracle.connid_counts."""
    f, d, od = family(name)
    sents = sentences(f)
    utf8, off = vb.Tokenizer.pack(sents)
    for isp, mgl in SETTINGS:
        e_off, e_toks, cnt = od.tokenize_batch(utf8, off, isp, mgl, want_counters=True)
        tok = tokenizer(d, "whole", isp, mgl)
        tok.set_counting(True)
        res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
        assert tok.describe()["last_viterbi"] == "k_viterbi"
        assert_same(res.tok_offsets, res.tokens, e_off, e_toks)
        np.testing.assert_array_equal(tok.last_counters(), cnt, err_msg=f"ignore_space={isp} mgl={mgl}")
    short = sentences(f, 80)
    for isp, mgl in ((False, 0), (True, 3)):
        tok = tokenizer(d, "whole", isp, mgl)
        tok.init_connid_counter()
        tok.tokenize_batch(short)
        lid, rid = tok.connid_counts()
        e_lid, e_rid = BoundedOracle(od, f.char_def, f.unk_def, isp, mgl).connid_counts([s.encode() for s in short])
        np.testing.assert_array_equal(lid, e_lid)
        np.testing.assert_array_equal(rid, e_rid)


def char_bounds(s, positions):
    """Byte offsets of the given character positions of s (those inside it)."""
    lb = lead_bytes(s.encode())
    return sorted({lb[p] for p in positions if 0 < p < len(lb) - 1})


@pytest.mark.parametrize("route", ["whole", "chunked", "device", "small"])
@pytest.mark.parametrize("name", cf.FAMILIES)
def test_bounded_calls(name, route):
    """Boundaries inside group runs, inside grouped space runs and at the 32-character chunk edges, against
    BoundedOracle."""
    f, d, od = family(name)
    sents = sentences(f, 520)
    rng = np.random.default_rng(5)
    bounds = []
    for i, s in enumerate(sents):
        pos = {1, 2, 31, 32, 33, 511, 512} if i % 2 else {int(x) for x in rng.integers(1, max(2, len(s)), 3)}
        pos |= {k + 1 for k, ch in enumerate(s) if ch in " xy﻿　" and i % 3 == 0}  # just past a space-class character
        bounds.append(char_bounds(s, pos))
    for isp, mgl in ((False, 0), (True, 0), (True, 3)):
        bo = BoundedOracle(od, f.char_def, f.unk_def, isp, mgl)
        tok = tokenizer(d, route, isp, mgl)
        for lo in range(0, len(sents), 40):
            part, pb = sents[lo:lo + 40], bounds[lo:lo + 40]
            e_off, e_toks = bo.tokenize_batch([s.encode() for s in part], pb)
            utf8, off = vb.Tokenizer.pack(part)
            if route == "device":
                import torch
                bo_off, bnd = vb.Tokenizer.pack_bounds(pb)
                d_utf8 = torch.from_numpy(utf8.copy()).cuda()
                d_off = torch.from_numpy(off.astype(np.int64)).cuda()
                d_bo = torch.from_numpy(bo_off.astype(np.int64)).cuda()
                d_bnd = torch.from_numpy(bnd.astype(np.int32) if len(bnd) else np.zeros(1, np.int32)).cuda()
                torch.cuda.synchronize()
                a, b, n = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), len(part), len(utf8),
                                                    d_bnd_offsets=d_bo.data_ptr(), d_bnd=d_bnd.data_ptr(), n_bnd=len(bnd))
                got = d2h(a, len(part) + 1, np.uint64), d2h(b, n, vb.TOKEN_DTYPE)
            else:
                res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=pb)
                got = res.tok_offsets, res.tokens
                if route == "small" and len(utf8) <= SMALL_BYTES:
                    assert tok.describe()["last_viterbi"] == "k_small_batch"
            assert_same(*got, e_off, e_toks, f"{route} ignore_space={isp} mgl={mgl} from {lo}")


SPAN_STARTS = "éー@\x00\U0001F600\U0010FFFF\U00010000漢ßpq"


@pytest.mark.parametrize("name", cf.FAMILIES)
def test_spans_at_class_edges(name):
    """Spans of 1-3 characters that start at multi-category, spilled, NUL and astral characters: where no lexicon
    word fits, the unknown word comes from the base category of the span's first character."""
    f, d, od = family(name)
    sents, spans = [], []
    for s in sentences(f, 80):
        sp, b, prev = [], lead_bytes(s.encode()), 0
        for k, ch in enumerate(s):
            if ch in SPAN_STARTS and b[k] >= prev and k + 1 < len(b):
                e = b[min(len(b) - 1, k + 1 + k % 3)]
                sp.append((b[k], e))
                prev = e
        if sp:
            sents.append(s)
            spans.append(sp)
    assert len(sents) > 20
    for mgl in (0, 3):
        so = SpanOracle(od, f.char_def, f.unk_def, False, mgl)
        e_off, e_toks = so.tokenize_batch([s.encode() for s in sents], [Constraints((), tuple(x)) for x in spans])
        tok = tokenizer(d, "whole", False, mgl)
        res = tok.tokenize_batch(sents, spans=spans)
        assert_same(res.tok_offsets, res.tokens, e_off, e_toks, f"mgl={mgl}")


def test_spans_and_secondary_space():
    """With ignore_space, a span that starts at a letter whose secondary category is SPACE is refused, and so is a
    span that the skip from such a letter runs into; a span after the skip's end is honoured.  The library has one
    message for every invalid span, so each refused call has a twin without ignore_space, which the same span passes:
    the refusal comes from the space skip and not from the span's shape."""
    f, d, od = family("multi")
    tok = tokenizer(d, "whole", True)
    plain = tokenizer(d, "whole", False)
    so = SpanOracle(od, f.char_def, f.unk_def, True)
    so_plain = SpanOracle(od, f.char_def, f.unk_def, False)
    # the first span starts at x; the skip from x (the run xabc) lands on 漢 at character 5, inside the second
    for sent, span, why in (("漢xab漢", (3, 5), "starts at a skipped space"), ("漢xabc漢字", (5, 10), "lands inside")):
        with pytest.raises(ValueError, match=why):
            so.tokenize_batch([sent.encode()], [Constraints((), (span,))])
        with pytest.raises(vb.VibratoError, match="not start at a space when ignore_space is on") as ei:
            tok.tokenize_batch([sent], spans=[[span]])
        assert ei.value.kind == "InvalidArgument"
        e_off, e_toks = so_plain.tokenize_batch([sent.encode()], [Constraints((), (span,))])
        res = plain.tokenize_batch([sent], spans=[[span]])
        assert_same(res.tok_offsets, res.tokens, e_off, e_toks, sent)
    sents, spans = ["漢xab漢字"], [[(6, 12)]]
    e_off, e_toks = so.tokenize_batch([s.encode() for s in sents], [Constraints((), tuple(spans[0]))])
    res = tok.tokenize_batch(sents, spans=spans)
    assert_same(res.tok_offsets, res.tokens, e_off, e_toks)


@pytest.mark.parametrize("name", ["multi", "spill"])
def test_marginals_lattice_uncertainty(name):
    """Marginals and the lattice (node for node) and uncertainty against their oracles at their usual tolerances."""
    f, d, od = family(name)
    sents = sentences(f, 70)
    for isp, mgl in ((False, 0), (True, 3)):
        bo = BoundedOracle(od, f.char_def, f.unk_def, isp, mgl)
        gl.check(bo, sents, gl.run(gl.make(d, isp=isp, mgl=mgl, theta=gl.THETA), "whole", sents), theta=gl.THETA)
        gu.check(bo, sents, gu.run(gu.make(d, isp=isp, mgl=mgl), "whole", sents))


@pytest.mark.parametrize("name", cf.FAMILIES)
def test_detail_text(name):
    f, d, od = family(name)
    sents = sentences(f)
    utf8, off = vb.Tokenizer.pack(sents)
    for isp in (False, True):
        tok_off, toks, _ = od.tokenize_batch(utf8, off, isp)
        tok = tokenizer(d, "whole", isp).output_mode("detail")
        text_off, text = tok.tokenize_batch(utf8=utf8, byte_offsets=off).text()
        e_off, e_text = vo.format_batch(od, utf8, off, tok_off, toks, "detail")
        assert text == e_text
        np.testing.assert_array_equal(text_off, e_off)


def test_refused_family():
    """A spilled base id with no unk.def slot: the tokenizer refuses the dictionary when it builds its device image
    (on first use), from readers and after a .dic round trip."""
    f = cf.make_family("refused")
    d = vb.SystemDictionaryBuilder.from_readers(*f.sources())
    for dic in (d, vb.Dictionary.read(d.write())):
        with pytest.raises(vb.VibratoError, match="CharInfo base_id has no unk.def slot") as ei:
            vb.Tokenizer.new(dic).tokenize_batch(["ab"])
        assert ei.value.kind == "BincodeDecode"


def test_category_without_unknown_words():
    """A category with no unk.def entry: a sentence whose lattice then has no path gets no tokens, as in the oracle;
    the other sentences of the batch are unaffected."""
    f = cf.make_family("multi")
    unk = "".join(line + "\n" for line in f.unk_def.splitlines() if not line.startswith("LATIN,"))
    lex = "".join(line + "\n" for line in f.lex_csv.splitlines() if "ß" not in line)
    src = (lex, f.matrix, f.char_def, unk)
    od = vo.OracleDictionary(*src)
    d = vb.SystemDictionaryBuilder.from_readers(*src)
    sents = ["abc", "aßb", "漢字", "ß", "ab ß", "x"]
    utf8, off = vb.Tokenizer.pack(sents)
    for isp in (False, True):
        e_off, e_toks, _ = od.tokenize_batch(utf8, off, isp)
        per = np.diff(e_off.astype(np.int64))
        assert per[1] == 0 and per[3] == 0 and per[0] > 0 and per[2] > 0
        for route in ("whole", "small", "device"):
            tok = tokenizer(d, route, isp)
            assert_same(*run_route(tok, route, sents), e_off, e_toks, f"{route} ignore_space={isp}")


# ---- UTF-8 ----

def invalid_sample(cases):
    """The invalid cases, sampled deterministically: for every lead byte 0x80-0xFF two 2-byte strings whose
    continuation values cycle through all of CONTINUATIONS, then every 1009th longer invalid string."""
    bad = [c for c in cases if not _valid(c)]
    two = [bytes([lead, cf.CONTINUATIONS[(3 * lead + k) % len(cf.CONTINUATIONS)]]) for lead in range(0x80, 0x100)
           for k in (0, 1)]
    longer = [c for c in bad if len(c) > 2][::1009]
    out = [c for c in two if not _valid(c)] + longer
    assert {c[0] for c in out} >= set(range(0x80, 0x100)) and {c[1] for c in out} >= set(cf.CONTINUATIONS)
    return out


def _valid(b):
    try:
        b.decode("utf-8")
        return True
    except UnicodeDecodeError:
        return False


def test_valid_utf8_batched():
    """Every valid string of the CPU set, as one batch, on the whole-batch and small-batch routes."""
    f, d, od = family("multi")
    good = [c for c in cf.utf8_cases() if _valid(c)]
    utf8, off = vb.Tokenizer.pack(good)
    e_off, e_toks, _ = od.tokenize_batch(utf8, off)
    tok = tokenizer(d, "whole")
    assert_same(*run_route(tok, "whole", good), e_off, e_toks)
    tok = tokenizer(d, "small")
    for batch in batches("small", good[:4000]):
        utf8, off = vb.Tokenizer.pack(batch)
        assert_same(*run_route(tok, "small", batch), *od.tokenize_batch(utf8, off)[:2])


UTF8_ROUTES = {
    "staged": ("whole", lambda bad: [b"ab", bad, b"cd"]),
    "unstaged": ("whole", lambda bad: [b"a" * 16400, bad]),
    "long_sentence": ("whole", lambda bad: [b"ab", "漢".encode() * 600 + bad]),
    "tile_last": ("whole", lambda bad: [b"ab"] * 31 + [bad] + [b"cd"] * 4),
    "small": ("small", lambda bad: [b"ab", bad, b"cd"]),
    "device": ("device", lambda bad: [b"ab", bad, b"cd"]),
}


@pytest.mark.parametrize("shape", list(UTF8_ROUTES))
def test_invalid_utf8_refused(shape):
    """Each sampled invalid string, one call each, is refused with kind Utf8; a good call after each one works."""
    route, build = UTF8_ROUTES[shape]
    f, d, od = family("multi")
    tok = tokenizer(d, route)
    good = ["ab漢\U0001F600", "x y"]
    utf8, off = vb.Tokenizer.pack(good)
    e_off, e_toks, _ = od.tokenize_batch(utf8, off)
    for bad in invalid_sample(cf.utf8_cases()):
        batch = build(bad)
        with pytest.raises(vb.VibratoError) as ei:
            run_route(tok, route, batch)
        assert ei.value.kind == "Utf8", bad.hex()
        assert_same(*run_route(tok, route, good), e_off, e_toks, bad.hex())
