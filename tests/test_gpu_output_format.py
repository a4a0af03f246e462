"""MeCab-style output formats (Tokenizer.output_format, `tokenize -F`), rendered on the device.

Text and text offsets are compared byte for byte with tests/format_oracle.py, a restatement of the directive table
in README.md over the oracle's tokens, on every host route: whole batch, chunked pipeline (with its retry when the
text outgrows its buffers), small_batch (with its fall-back) and multi-device."""
import os
import subprocess

import numpy as np
import pytest

import adversarial as adv
import format_oracle as fo
import vibrato_b200 as vb
from vibrato_b200 import synth
from oracle import vibrato_oracle as vo
from test_gpu_marginals import shard_devices

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (node, unk, bos, eos): every directive, fields with and without an unk format of their own
FORMATS = [
    ("%m\\t%M|%pS|%H|%f[6]|%f[0,1,2,30]|%F,[5,0]|%F\\s[1,6]\\n", "U:%m\\t%f[0,3,6]\\t%s\\n", "B%L:", "E%S\\n"),
    ("%m %c %pw %pc %pn %pC %ps %pe %pl %pL %phl %phr %s %%\\n", None, "", "EOS\\n"),
    ("%f[6] ", None, "", "\\n"),
    ("%m\\t%f[0,1]\\t%pc\\t%pC\\n", "%m\\t%f[0,1]\\t%pc\\t%pC\\t*\\n", "\\s\\t", "%L\\a\\b\\v\\f\\r\\0\\\\EOS\\n"),
]


def assert_text(res, off, text):
    toff, got = res.text()
    np.testing.assert_array_equal(toff, off)
    assert got == text


def chunk_bounds(n_sent, chunk):
    """The chunk plan of the host pipeline (engine.cu run_host)."""
    lo = max(1024, chunk // 2)
    bounds = [0, min(n_sent, lo)]
    while bounds[-1] < n_sent:
        rest = n_sent - bounds[-1]
        bounds.append(bounds[-1] + (rest if rest <= lo + lo // 2 else max(lo, rest // 2)))
    return bounds


def empty_runs(off, centres, k=3):
    """Sentences around every centre become empty (their bytes join a neighbour)."""
    off = off.copy()
    for c in centres:
        off[c - k + 1:c + k + 1] = off[c - k + 1]
    return off


class Synth:
    """synth-small with a user lexicon and two quoted-feature rows, on the device and in the oracle."""

    def __init__(self):
        sd = synth.make_dictionary("synth-small")
        lex = sd.lex_csv + '"ｘ,ｙ",3,3,-900,記号,"x""y",*,"p,q",,*z\n'.encode()
        self.user = synth.make_user_csv(sd, 500)
        self.sd = sd
        self.d = vb.SystemDictionaryBuilder.from_readers(lex, sd.matrix, sd.char_def, sd.unk_def)
        self.d.reset_user_lexicon_from_reader(self.user)
        self.od = vo.OracleDictionary(lex, sd.matrix, sd.char_def, sd.unk_def).set_user_csv(self.user)

    def corpus(self, n, seed):
        utf8, off = synth.make_corpus(self.sd, n, seed=seed, log_uniform=(1, 200), unk_frac=0.15, space_frac=0.04,
                                      user_csv=self.user, user_frac=0.05)
        extra = ["１,２ｘ,ｙ１,２", " ｘ,ｙ  ｘ,ｙ ", "", "   ", "ｘ,ｙ"]
        u2, o2 = vb.Tokenizer.pack(extra)
        return np.concatenate([utf8, u2]), np.concatenate([off, o2[1:] + off[-1]]).astype(np.uint64)


@pytest.fixture(scope="module")
def syn():
    return Synth()


def expected(od, fmt, utf8, off, ignore_space=False, mgl=0):
    tok_off, toks = od.tokenize_batch(utf8, off, ignore_space, mgl, n_threads=8)[:2]
    return fo.format_batch(od, fo.Format(*fmt), utf8, off, tok_off, toks)


@pytest.mark.parametrize("ignore_space", [False, True])
@pytest.mark.parametrize("mgl", [0, 3])
def test_every_directive_whole_batch(syn, ignore_space, mgl):
    utf8, off = syn.corpus(3000, seed=11)
    tok = vb.Tokenizer.new(syn.d).ignore_space(ignore_space).max_grouping_len(mgl)
    tok.set_option("chunk_sentences", 0)
    for fmt in FORMATS:
        eoff, etext = expected(syn.od, fmt, utf8, off, ignore_space, mgl)
        assert_text(tok.output_format(*fmt).tokenize_batch(utf8=utf8, byte_offsets=off), eoff, etext)
    if not ignore_space and mgl == 0:  # the restatement itself: skipped fields, quotes, unknown words' short features
        _, etext = expected(syn.od, FORMATS[0], utf8, off)
        assert b'\tx"y|' in etext and b"U:" in etext and b"|*" not in etext


def test_mecab_format_equals_mecab_mode(syn):
    utf8, off = syn.corpus(2000, seed=5)
    tok = vb.Tokenizer.new(syn.d).ignore_space(True)
    a = tok.output_mode("mecab").tokenize_batch(utf8=utf8, byte_offsets=off).text()
    b = tok.output_format("%m\t%H\n").tokenize_batch(utf8=utf8, byte_offsets=off).text()
    np.testing.assert_array_equal(a[0], b[0])
    assert a[1] == b[1]


@pytest.mark.parametrize("chunk,dual", [(256, 0), (1024, 1)])
def test_chunked_with_empty_runs_at_chunk_boundaries(syn, chunk, dual):
    utf8, off = syn.corpus(4000, seed=31)
    n = len(off) - 1
    bounds = chunk_bounds(n, chunk)
    assert len(bounds) > 3
    off = empty_runs(off, bounds[1:-1]).astype(np.uint64)
    off = np.concatenate([off, [off[-1]] * 5]).astype(np.uint64)
    tok = vb.Tokenizer.new(syn.d).ignore_space(True)
    tok.set_option("chunk_sentences", chunk)
    tok.set_option("dual_stream", dual)
    for fmt in FORMATS:
        eoff, etext = expected(syn.od, fmt, utf8, off, True)
        tok.output_format(*fmt)
        for _ in range(2):  # the second call reuses the buffers and the learned text ratio
            assert_text(tok.tokenize_batch(utf8=utf8, byte_offsets=off), eoff, etext)


def test_chunked_text_overflow_retry(syn):
    """%S per token: far more text per input byte than a fresh format's buffers are sized for."""
    utf8, off = syn.corpus(3000, seed=8)
    fmt = ("%S\\t%m\\n", None, "", "EOS\\n")
    eoff, etext = expected(syn.od, fmt, utf8, off)
    assert len(etext) > 20 * len(utf8)
    tok = vb.Tokenizer.new(syn.d)
    tok.set_option("chunk_sentences", 256)
    tok.output_format(*fmt)
    for _ in range(2):
        assert_text(tok.tokenize_batch(utf8=utf8, byte_offsets=off), eoff, etext)


def test_small_batch_and_its_fallback(syn):
    utf8, off = syn.corpus(400, seed=3)
    tok = vb.Tokenizer.new(syn.d).ignore_space(True).small_batch(64)
    for fmt in FORMATS:
        tok.output_format(*fmt)
        for s in range(0, 400, 64):
            e = min(s + 64, len(off) - 1)
            o = (off[s:e + 1] - off[s]).astype(np.uint64)
            u = utf8[int(off[s]):int(off[e])]
            eoff, etext = expected(syn.od, fmt, u, o, True)
            assert_text(tok.tokenize_batch(utf8=u, byte_offsets=o), eoff, etext)
            assert tok.describe()["last_viterbi"] == "k_small_batch"
    # more than the route's 2 MiB of text: the batch runs again on the usual route, with the same text
    sents = ["ｘ,ｙ" * 600] * 3
    u, o = vb.Tokenizer.pack(sents)
    fmt = ("%S%S%S%S\\n", None, "", "EOS\\n")
    eoff, etext = expected(syn.od, fmt, u, o, True)
    assert len(etext) > (2 << 20)
    assert_text(tok.output_format(*fmt).tokenize_batch(utf8=u, byte_offsets=o), eoff, etext)
    assert tok.describe()["last_viterbi"] != "k_small_batch"


@pytest.mark.parametrize("family,connector", [("ties", "matrix"), ("extreme", "matrix"), ("wrap", "raw"),
                                              ("wrap", "dual")])
def test_adversarial_costs_and_connectors(family, connector):
    d = adv.make_dictionary(family, dual=connector == "dual")
    if connector == "matrix":
        dev = vb.SystemDictionaryBuilder.from_readers(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    else:
        right, left, cost = d.matrix
        dev = vb.SystemDictionaryBuilder.from_readers_with_bigram_info(d.lex_csv, right, left, cost, d.char_def,
                                                                       d.unk_def, dual_connector=connector == "dual")
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def, dual_connector=connector == "dual")
    dev.reset_user_lexicon_from_reader(d.user_csv)
    od.set_user_csv(d.user_csv)
    utf8, off = adv.pack(adv.make_sentences(d, 600, seed=4))
    fmt = ("%m %c %pc %pn %pC %pL %phl %phr %s %f[0,1]\\n", None, "[%L]", "EOS\\n")
    for ignore_space in (False, True):
        tok = vb.Tokenizer.new(dev).ignore_space(ignore_space).output_format(*fmt)
        eoff, etext = expected(od, fmt, utf8, off, ignore_space)
        assert_text(tok.tokenize_batch(utf8=utf8, byte_offsets=off), eoff, etext)
    # empty batch, empty sentences
    for sents in ([], ["", ""]):
        u, o = vb.Tokenizer.pack(sents)
        eoff, etext = expected(od, fmt, u, o)
        assert_text(tok.tokenize_batch(utf8=u, byte_offsets=o), eoff, etext)


def test_switching_and_rebuild(syn):
    utf8, off = syn.corpus(500, seed=9)
    tok = vb.Tokenizer.new(syn.d)
    fmt = FORMATS[0]
    eoff, etext = expected(syn.od, fmt, utf8, off)
    assert_text(tok.output_format(*fmt).tokenize_batch(utf8=utf8, byte_offsets=off), eoff, etext)
    tok_off, toks = syn.od.tokenize_batch(utf8, off)[:2]
    moff, mtext = vo.format_batch(syn.od, utf8, off, tok_off, toks, "wakati")
    assert_text(tok.output_mode("wakati").tokenize_batch(utf8=utf8, byte_offsets=off), moff, mtext)
    assert_text(tok.output_format(*fmt).tokenize_batch(utf8=utf8, byte_offsets=off), eoff, etext)
    # a format set before ignore_space() survives the rebuilt engine
    tok.ignore_space(True)
    eoff2, etext2 = expected(syn.od, fmt, utf8, off, True)
    assert_text(tok.tokenize_batch(utf8=utf8, byte_offsets=off), eoff2, etext2)
    assert "field_table" in tok.describe()
    tok.output_format(None)
    with pytest.raises(vb.VibratoError):
        tok.tokenize_batch(utf8=utf8, byte_offsets=off).text()
    tok.output_mode("wakati").output_format(None)  # switching a format off leaves a fixed mode alone
    assert_text(tok.tokenize_batch(utf8=utf8, byte_offsets=off), *vo.format_batch(
        syn.od, utf8, off, *syn.od.tokenize_batch(utf8, off, True)[:2], "wakati"))


BAD = [
    ("%h", 0, "%h"), ("ab%t", 2, "%t"), ("%P", 0, "%P"), ("x%pP", 1, "%pP"), ("%pA", 0, "%pA"), ("%pB", 0, "%pB"),
    ("%pi", 0, "%pi"), ("%pb", 0, "%pb"), ("%m%pp", 2, "%pp"), ("%q", 0, "%q"), ("%phx", 0, "%ph"),
    ("%f", 0, "%f"), ("%f[", 0, "%f"), ("%f[1,]", 0, "%f"), ("%f[a]", 0, "%f"), ("%F", 0, "%F"), ("%F,", 0, "%F"),
    ("%f[256]", 0, "%f"), ("\\q", 0, "\\q"), ("abc%", 3, "'%'"),
    ("%f[0,1,2,3,4,5,6,7]%F,[8,9,10,11,12,13,14,15,16]", 19, "%F"),
]


@pytest.mark.parametrize("node,pos,what", BAD)
def test_compile_errors(syn, node, pos, what):
    tok = vb.Tokenizer.new(syn.d)
    with pytest.raises(vb.VibratoError) as e:
        tok.output_format(node)
    assert e.value.kind == "InvalidArgument"
    assert f"byte {pos}" in str(e.value) and what in str(e.value), str(e.value)
    with pytest.raises(fo.FormatError):  # the restatement rejects it too
        fo.Format(node)


def test_bos_eos_and_compact_are_refused(syn):
    tok = vb.Tokenizer.new(syn.d)
    for bos, eos, pos, what in (("%m", "", 0, "%m"), ("", "EOS%H", 3, "%H"), ("", "%f[1]", 0, "%f")):
        with pytest.raises(vb.VibratoError) as e:
            tok.output_format("%m", None, bos, eos)
        assert f"byte {pos}" in str(e.value) and what in str(e.value)
    with pytest.raises(vb.VibratoError):
        vb.Tokenizer.new(syn.d).output_format("%m").compact_tokens(True)
    with pytest.raises(vb.VibratoError):
        vb.Tokenizer.new(syn.d).compact_tokens(True).output_format("%m")


def test_text_too_large_for_the_device_is_an_error():
    """%S 200 times per token over a 64 KiB sentence of one-byte tokens: about 860 GB of text."""
    lex, matrix, char_def, unk_def = adv.single_word_dictionary(0, 0)
    tok = vb.Tokenizer.new(vb.SystemDictionaryBuilder.from_readers(lex, matrix, char_def, unk_def))
    tok.set_option("chunk_sentences", 0)
    tok.output_format("%S" * 200)
    with pytest.raises(vb.VibratoError):
        tok.tokenize_batch(["a" * 65536])
    tok.output_format("%m,")
    _, text = tok.tokenize_batch(["aaa"]).text()
    assert text == b"a,a,a,EOS\n"


def test_multi_device(syn):
    utf8, off = syn.corpus(3000, seed=21)
    multi = vb.Tokenizer.new(syn.d, devices=shard_devices(2)).ignore_space(True)
    for fmt in FORMATS:
        eoff, etext = expected(syn.od, fmt, utf8, off, True)
        assert_text(multi.output_format(*fmt).tokenize_batch(utf8=utf8, byte_offsets=off), eoff, etext)
    for sents in (["ｘ,ｙ"], ["", "", ""], []):
        u, o = vb.Tokenizer.pack(sents)
        assert_text(multi.tokenize_batch(utf8=u, byte_offsets=o), *expected(syn.od, FORMATS[-1], u, o, True))


def test_tokenize_cli(golden, tmp_path):
    exe = os.path.join(ROOT, "vibrato_b200", "bin", "tokenize")
    if not os.path.exists(exe):
        pytest.skip("CLIs not built")
    r = golden["resources"]
    for k, v in r.items():
        (tmp_path / k).write_text(v, encoding="utf-8", newline="")
    lines = ["京都東京都京都", "東京 都", "", "kampersanda", "東京県に行く"] * 3
    data = ("\n".join(lines) + "\n").encode()
    node, unk, eos = "%m/%f[0]/%pC ", "?%m ", "\\n"
    d = vb.SystemDictionaryBuilder.from_readers(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
    d.reset_user_lexicon_from_reader(r["user.csv"])
    tok = vb.Tokenizer.new(d).ignore_space(True).output_format(node, unk, "", eos)
    _, want = tok.tokenize_batch(lines).text()
    base = [exe, "-i", str(tmp_path), "-u", str(tmp_path / "user.csv"), "-S"]
    for flags in ([], ["--batch-lines", "1"], ["-O", "wakati"]):  # -F takes precedence over -O
        p = subprocess.run(base + ["-F", node, "--unk-format", unk, "--eos-format", eos] + flags, input=data,
                           capture_output=True, timeout=120)
        assert p.returncode == 0, p.stderr.decode()
        assert p.stdout == want
    p = subprocess.run(base + ["-F", node, "--format-on", "host"], input=data, capture_output=True, timeout=120)
    assert p.returncode == 2
    p = subprocess.run(base + ["-F", "%pP"], input=data, capture_output=True, timeout=120)
    assert p.returncode == 1 and b"%pP" in p.stderr
