"""Sample text on the GPU (option "sample_text" = 1): the output text renders each sentence's n samples, in order, in
place of its best path.  The text is pinned to the result's own sample records by the restatements the output-stage
tests use (the records themselves are pinned to tests/sampling_oracle.py by test_gpu_sampling.py); it is
byte-identical on every route, a sample on the best path renders to the sentence's best-path text, and nothing else
changes.  Also "sample_base", the refusals, and `tokenize --sample`."""
import os
import subprocess

import numpy as np
import pytest

import adversarial as adv
import format_oracle as fo
import vibrato_b200 as vb
from test_gpu_marginals import adversarial_dicts, golden_dicts, golden_sents, shard_devices, shard_devices_arg
from vibrato_b200 import VibratoError
from oracle import vibrato_oracle as vo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THETA = 0.01
MODES = ("mecab", "wakati", "detail")
FORMATS = [
    ("%m ", None, "", "\n"),
    ("%f[6] ", None, "", "\n"),
    ("%m\t%f[0,1]\t%pc\t%pC\n", "%m\t?\t%pc\t%pn\n", "", "EOS\n"),
    ("[%M|%pS|%pn|%pL]", None, "", "\n"),  # the "prev" directives: the previous record of the same sample
    ("%m/%ps-%pe ", None, "BOS %L <%S>\n", "\nEOS %L\n"),
]


def style_of(tok, style):
    """Sets an output mode (str) or format (tuple) on tok."""
    return tok.output_mode(style) if isinstance(style, str) else tok.output_format(*style)


def call(tok, sents, bounds=None):
    """(text_offsets, text, sample_offsets, samples, tok_offsets, tokens) of one host call."""
    res = tok.tokenize_batch(sents, boundaries=bounds)
    toff, text = res.text()
    out = (toff, text) + tuple(None if x is None else x.copy()
                               for x in (res.sample_offsets, res.samples, res.tok_offsets, res.tokens))
    res.close()
    return out


def restated(od, style, sents, n, sample_off, samples):
    """(text_offsets, text) the restatement gives for the samples: every sentence repeated n times, walk s * n + j
    rendered as a sentence whose tokens are sample j's records; a sentence's text starts at its first walk."""
    utf8, off = vb.Tokenizer.pack([s for s in sents for _ in range(n)])
    if isinstance(style, str):
        woff, text = vo.format_batch(od, utf8, off, sample_off, samples, style)
    else:
        woff, text = fo.format_batch(od, fo.Format(*style), utf8, off, sample_off, samples)
    return np.asarray(woff, dtype=np.uint64)[::n], text


def check_restated(tok, od, style, sents, n, bounds=None):
    toff, text, soff, samples, _, _ = call(style_of(tok, style), sents, bounds)
    assert len(toff) == len(sents) + 1 and len(soff) == len(sents) * n + 1
    eoff, etext = restated(od, style, sents, n, soff, samples)
    assert text == etext, style
    np.testing.assert_array_equal(toff, eoff)


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("seed", [0, 2 ** 64 - 1])
def test_text_equals_restatement_golden(golden, n, seed):
    sents = golden_sents(golden) + ["東京都に行った。", "あ", "京都 東京"]
    d, od, _ = golden_dicts(golden, True)
    for isp in (False, True):
        tok = vb.Tokenizer.new(d).ignore_space(isp).sampling(n, THETA, seed, text=True)
        for style in MODES + tuple(FORMATS):
            check_restated(tok, od, style, sents, n)


@pytest.mark.parametrize("family", list(adv.FAMILIES) + ["raw", "dual"])
def test_text_equals_restatement_adversarial(family):
    d, dev, od = adversarial_dicts(family)
    sents = adv.make_sentences(d, 30, seed=5, max_len=40) + [" ", "a  ", ""]
    theta = 0.05 if family in adv.FAMILIES else 1e-6  # the wrap family's costs are near +-2^31
    tok = vb.Tokenizer.new(dev).ignore_space(True).sampling(3, theta, 7, text=True)
    for style in ("mecab", "detail", FORMATS[2], FORMATS[3]):
        check_restated(tok, od, style, sents, 3)


def test_text_equals_restatement_bounded(golden):
    d, od, _ = golden_dicts(golden, False)
    sents = ["京都東京都京都", "アイアイウ", "東京   都", ""] * 5
    bounds = [[12], [6], [], []] * 5
    tok = vb.Tokenizer.new(d).ignore_space(True).sampling(3, THETA, 1, text=True)
    for style in ("mecab", FORMATS[3]):
        check_restated(tok, od, style, sents, 3, bounds)


def long_feature_dict():
    """One-character surfaces with 1-2 KB features: a fresh tokenizer's chunk text buffers overflow (the retry)."""
    rng = np.random.default_rng(8)
    chars = "abcdefghijklmnop"
    lex = "".join(f"{c},0,0,{10 * i},{c}:" + "x" * int(rng.integers(1000, 2000)) + "\n" for i, c in enumerate(chars))
    matrix, char_def, unk_def = "1 1\n0 0 0\n", "DEFAULT 0 1 0\n", "DEFAULT,0,0,30000,*\n"
    d = vb.SystemDictionaryBuilder.from_readers(lex, matrix, char_def, unk_def)
    od = vo.OracleDictionary(lex, matrix, char_def, unk_def)
    sents = ["".join(rng.choice(list(chars), size=int(rng.integers(0, 30)))) for _ in range(1500)]
    return d, od, sents


@pytest.mark.parametrize("route", ["chunked", "retry", "multi"])
def test_routes_are_byte_identical(golden, route):
    if route == "retry":
        d, od, sents = long_feature_dict()
        styles = ("mecab", "detail")
    else:
        d, od, _ = golden_dicts(golden, True)
        sents = (golden_sents(golden) + ["東京都に行った。", "京都 東京"]) * 40
        styles = MODES + (FORMATS[3], FORMATS[4])
    for style in styles:
        ref = call(style_of(vb.Tokenizer.new(d).sampling(3, THETA, 5, text=True), style), sents)
        tok = vb.Tokenizer.new(d, devices=shard_devices(2)) if route == "multi" else vb.Tokenizer.new(d)
        if route != "multi":
            tok.set_option("chunk_sentences", 64 if route == "chunked" else 256)
        style_of(tok.sampling(3, THETA, 5, text=True), style)
        for _ in range(2):  # the second call runs with the ratios the first one learned
            got = call(tok, sents)
            assert got[1] == ref[1], (route, style)
            for a, b in zip(got[:1] + got[2:], ref[:1] + ref[2:]):
                assert a.tobytes() == b.tobytes(), (route, style)
        if route == "retry":
            eoff, etext = restated(od, style, sents, 3, ref[2], ref[3])
            assert ref[1] == etext and len(etext) > 500 * sum(len(s) for s in sents)


def test_sample_on_the_best_path_renders_the_best_path_text(golden):
    d, od, _ = golden_dicts(golden, True)
    sents = golden_sents(golden) + ["東京都に行った。", "京都 東京"]
    hits = 0
    for style in MODES + tuple(FORMATS):
        best = call(style_of(vb.Tokenizer.new(d), style), sents)
        samp = call(style_of(vb.Tokenizer.new(d).sampling(4, 0.5, 3, text=True), style), sents)
        _, btext, _, _, bto, btoks = best
        _, stext, soff, samples, _, _ = samp
        utf8, off = vb.Tokenizer.pack([s for s in sents for _ in range(4)])
        woff = vo.format_batch(od, utf8, off, soff, samples, style)[0] if isinstance(style, str) else \
            fo.format_batch(od, fo.Format(*style), utf8, off, soff, samples)[0]
        for i in range(len(sents)):
            tokens = btoks[int(bto[i]):int(bto[i + 1])].tobytes()
            for j in range(4):
                w = i * 4 + j
                if samples[int(soff[w]):int(soff[w + 1])].tobytes() != tokens:
                    continue
                hits += 1
                from_best = btext[int(best[0][i]):int(best[0][i + 1])]
                assert stext[int(woff[w]):int(woff[w + 1])] == from_best, (style, i, j)
    assert hits > 50


def test_nothing_else_changes(golden):
    d, od, _ = golden_dicts(golden, True)
    sents = golden_sents(golden) * 3
    for style in ("mecab", FORMATS[2]):
        outs = []
        for text in (False, True):
            tok = vb.Tokenizer.new(d).marginals(THETA).lattice(True).sampling(3, THETA, 9, text=text)
            res = style_of(tok, style).tokenize_batch(sents)
            outs.append([res.tok_offsets.copy(), res.tokens.copy(), res.token_probs.copy(), res.path_probs.copy(),
                         res.sample_offsets.copy(), res.samples.copy(), res.node_offsets.copy(), res.nodes.copy(),
                         res.node_links.copy(), res.node_probs.copy(), res.text()])
            res.close()
        for a, b in zip(outs[0][:-1], outs[1][:-1]):
            assert a.tobytes() == b.tobytes()
        # the token text with sampling on and sample text off is the text with sampling off
        plain = call(style_of(vb.Tokenizer.new(d).marginals(THETA).lattice(True), style), sents)
        assert outs[0][-1][1] == plain[1]
        np.testing.assert_array_equal(outs[0][-1][0], plain[0])


def test_sample_base(golden):
    d, od, _ = golden_dicts(golden, True)
    pool = golden_sents(golden) + ["東京都に行った。", "京都 東京"]
    sents = [pool[i % len(pool)] for i in range(200)]
    whole = call(vb.Tokenizer.new(d).sampling(3, THETA, 11, text=True).output_mode("wakati"), sents)
    tok = vb.Tokenizer.new(d).sampling(3, THETA, 11, text=True).output_mode("wakati")
    text, samples = b"", []
    for a, b in ((0, 70), (70, 150), (150, 200)):
        part = call(tok.sample_base(a), sents[a:b])
        text += part[1]
        samples.append(part[3])
    assert text == whole[1]
    assert np.concatenate(samples).tobytes() == whole[3].tobytes()
    base0 = call(vb.Tokenizer.new(d).sampling(3, THETA, 11, text=True).output_mode("wakati").sample_base(0), sents)
    assert base0[1] == whole[1] and base0[3].tobytes() == whole[3].tobytes()
    assert call(tok.sample_base(2 ** 32 - 200), sents)[1].count(b"\n") == 3 * len(sents)  # the last index fits
    tok.sample_base(2 ** 32 - 199)
    with pytest.raises(VibratoError, match="sample_base"):
        tok.tokenize_batch(sents)
    with pytest.raises(VibratoError, match="sample_base"):
        tok.sample_base(-1)


def test_refusals_and_replay(golden):
    d, od, _ = golden_dicts(golden, True)
    tok = vb.Tokenizer.new(d)
    with pytest.raises(VibratoError, match="needs sampling"):
        tok.set_option("sample_text", 1)
    tok.sampling(2, THETA, 1, text=True)
    with pytest.raises(VibratoError, match="sample_text"):
        tok.set_option("sample_text", 2)
    with pytest.raises(VibratoError, match="switching sampling off"):
        lib_set_sampling(tok, 0)  # Tokenizer.sampling(0) would switch sample text off first
    with pytest.raises(VibratoError, match="lattice"):
        tok.lattice(True, text=True)
    # %pP and %pb, in either order, named with their byte position
    tok.marginals(THETA)
    with pytest.raises(VibratoError, match=r"node format, byte 3: %pP has no value in sample text"):
        tok.output_format("%m\t%pP\n")
    with pytest.raises(VibratoError, match=r"node format, byte 2: %pb has no value in sample text"):
        tok.output_format("%m%pb\n")
    tok.sampling(2, THETA, 1, text=False)
    tok.output_format("%m\t%pP\n")
    with pytest.raises(VibratoError, match=r"node format, byte 3: %pP has no value in sample text"):
        tok.set_option("sample_text", 1)
    tok.output_mode("wakati").lattice(True, text=True)
    with pytest.raises(VibratoError, match="lattice"):
        tok.set_option("sample_text", 1)
    # sample text survives the engine's rebuild
    sents = golden_sents(golden)
    tok = vb.Tokenizer.new(d).sampling(3, THETA, 4, text=True).output_format(*FORMATS[3])
    before = call(tok, sents)
    tok.ignore_space(False)
    after = call(tok, sents)
    assert after[1] == before[1] and after[0].tobytes() == before[0].tobytes()


def lib_set_sampling(tok, n):
    from vibrato_b200._native import lib
    from vibrato_b200.api import check
    check(lib().vbt_tokenizer_set_sampling(tok.handle(), n, THETA, 1))


def test_tokenize_cli_sample(golden, tmp_path):
    exe = os.path.join(ROOT, "vibrato_b200", "bin", "tokenize")
    if not os.path.exists(exe):
        pytest.skip("CLIs not built")
    for k, v in golden["resources"].items():
        (tmp_path / k).write_text(v, encoding="utf-8", newline="")
    lines = ["京都東京都京都", "東京 都", "", "kampersanda", "東京県に行く", "", "京都 東京"] * 3
    text = ("\n".join(lines) + "\n").encode()
    d, od, _ = golden_dicts(golden, True)
    base = [exe, "-i", str(tmp_path), "-u", str(tmp_path / "user.csv"), "--sample", "3", "-t", "0.01", "--seed", "5"]
    flag_sets = [["--batch-lines", "1"], ["--batch-lines", "7"], ["--batch-lines", "65536"], ["--devices", "0"]]
    flag_sets += [["--devices", shard_devices_arg(2)], ["--devices", shard_devices_arg(2), "--batch-lines", "7"]]
    for style, flags in (("wakati", ["-O", "wakati"]), (FORMATS[3], ["-F", FORMATS[3][0], "--eos-format", "\n"])):
        tok = style_of(vb.Tokenizer.new(d).sampling(3, 0.01, 5, text=True), style)
        expected = call(tok, lines)[1]
        for extra in flag_sets:
            p = subprocess.run(base + flags + extra, input=text, capture_output=True, timeout=120)
            assert p.returncode == 0, p.stderr.decode()
            assert p.stdout == expected, (style, extra)
    # --boundary-marker: the marker's boundaries, whatever the batch
    marked = ["京都|東京都京都", "東京 都", "", "東京|県に行く"] * 3
    mtext = ("\n".join(marked) + "\n").encode()
    sents = [s.replace("|", "") for s in marked]
    bounds = [[s.encode().index(b"|")] if "|" in s else [] for s in marked]
    expected = call(vb.Tokenizer.new(d).sampling(3, 0.01, 5, text=True).output_mode("wakati"), sents, bounds)[1]
    for extra in flag_sets[:3]:
        p = subprocess.run(base + ["-O", "wakati", "--boundary-marker", "|"] + extra, input=mtext, capture_output=True,
                           timeout=120)
        assert p.returncode == 0, p.stderr.decode()
        assert p.stdout == expected, extra
    assert expected.count(b"\n") == 3 * len(marked)
