"""The output stage (Tokenizer.output_mode, BatchResult.text) on every host route: the chunked host pipeline, its
retry when the text outgrows the buffer sized for it, multi-device tokenizers and the `tokenize` CLI flags that
reach them.  Text and text offsets are compared with the oracle's rendering of its own tokens and with the
single-device whole-batch route, byte for byte."""
import os
import subprocess

import numpy as np
import pytest

import vibrato_b200 as vb
from vibrato_b200 import synth
from oracle import vibrato_oracle as vo
from test_gpu_marginals import shard_devices, shard_devices_arg

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("mecab", "wakati", "detail")


def assert_batch_equal(res, tok_off, toks):
    assert res.n_sent == len(tok_off) - 1
    np.testing.assert_array_equal(res.tok_offsets, tok_off)
    assert res.n_tokens == len(toks)
    for name in vb.TOKEN_DTYPE.names:
        np.testing.assert_array_equal(res.tokens[name], toks[name], err_msg=name)


def assert_text_equal(res, off, text):
    toff, got = res.text()
    np.testing.assert_array_equal(toff, off)
    assert got == text


def chunk_bounds(n_sent, chunk):
    """The chunk plan of the host pipeline (engine.cu run_host): where one chunk ends and the next begins."""
    lo = max(1024, chunk // 2)
    bounds = [0, min(n_sent, lo)]
    while bounds[-1] < n_sent:
        rest = n_sent - bounds[-1]
        bounds.append(bounds[-1] + (rest if rest <= lo + lo // 2 else max(lo, rest // 2)))
    return bounds


def empty_around(off, centres, k=3):
    """Sentences centre-k+1 .. centre+k-1 become empty; their bytes join sentence centre+k (still valid UTF-8)."""
    off = off.copy()
    for c in centres:
        off[c - k + 1:c + k + 1] = off[c - k + 1]
    return off


def synth_user_dictionary():
    sd = synth.make_dictionary("synth-small")
    user = synth.make_user_csv(sd, 500)
    d = vb.SystemDictionaryBuilder.from_readers(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
    d.reset_user_lexicon_from_reader(user)
    od = vo.OracleDictionary(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
    od.set_user_csv(user)
    return sd, user, d, od


@pytest.mark.parametrize("chunk", [256, 1024])
@pytest.mark.parametrize("dual", [0, 1])
def test_chunked_text_matches_oracle_and_whole_batch(chunk, dual):
    sd, user, d, od = synth_user_dictionary()
    n = 4000
    utf8, off = synth.make_corpus(sd, n, seed=31, log_uniform=(1, 300), unk_frac=0.15, space_frac=0.03, user_csv=user,
                                  user_frac=0.05)
    bounds = chunk_bounds(n, chunk)
    assert len(bounds) > 3
    off = empty_around(off, bounds[1:-1]).astype(np.uint64)  # runs of empty sentences across every chunk boundary
    off = np.concatenate([off, [off[-1]] * 5]).astype(np.uint64)  # and at the very end
    tok_off, toks = od.tokenize_batch(utf8, off, True, n_threads=8)[:2]
    counts = np.diff(tok_off.astype(np.int64))
    assert counts.max() > 32 and all(counts[b - 1:b + 1].sum() == 0 for b in bounds[1:-1])
    whole = vb.Tokenizer.new(d).ignore_space(True)
    whole.set_option("chunk_sentences", 0)
    tok = vb.Tokenizer.new(d).ignore_space(True)
    tok.set_option("chunk_sentences", chunk)
    tok.set_option("dual_stream", dual)
    for mode in MODES:
        eoff, etext = vo.format_batch(od, utf8, off, tok_off, toks, mode)
        ref = whole.output_mode(mode).tokenize_batch(utf8=utf8, byte_offsets=off)
        assert_text_equal(ref, eoff, etext)
        for _ in range(2):  # the second call reuses the slots' buffers and the pinned result pool
            res = tok.output_mode(mode).tokenize_batch(utf8=utf8, byte_offsets=off)
            assert_batch_equal(res, tok_off, toks)
            assert_text_equal(res, eoff, etext)
    tok.output_mode(None)
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
    assert_batch_equal(res, tok_off, toks)
    with pytest.raises(vb.VibratoError):
        res.text()


def test_chunked_text_retry_when_the_text_outgrows_its_buffer():
    """One-character surfaces with 1-2 KB features: far more text per input byte than the pipeline sizes its text
    buffers for on a fresh tokenizer, so chunks overflow them and the batch is re-run with the measured ratio."""
    rng = np.random.default_rng(8)
    chars = "abcdefghijklmnop"
    lex = "".join(f"{c},0,0,{10 * i},{c}:" + "x" * int(rng.integers(1000, 2000)) + "\n" for i, c in enumerate(chars))
    matrix, char_def, unk_def = "1 1\n0 0 0\n", "DEFAULT 0 1 0\n", "DEFAULT,0,0,30000,*\n"
    d = vb.SystemDictionaryBuilder.from_readers(lex, matrix, char_def, unk_def)
    od = vo.OracleDictionary(lex, matrix, char_def, unk_def)
    sents = ["".join(rng.choice(list(chars), size=int(rng.integers(0, 30)))) for _ in range(3000)]
    utf8, off = vb.Tokenizer.pack(sents)
    tok_off, toks = od.tokenize_batch(utf8, off)[:2]
    for mode in ("mecab", "detail"):
        eoff, etext = vo.format_batch(od, utf8, off, tok_off, toks, mode)
        assert len(etext) > 500 * len(utf8)
        tok = vb.Tokenizer.new(d).output_mode(mode)
        tok.set_option("chunk_sentences", 256)
        tok.init_connid_counter()
        for _ in range(2):
            res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
            assert_batch_equal(res, tok_off, toks)
            assert_text_equal(res, eoff, etext)
        # the attempts that overflowed left no connection-id counts behind: two batches' worth, as without retries
        lid, rid = tok.connid_counts()
        olid, orid = od.connid_counts(utf8, off, False, n_threads=8)
        np.testing.assert_array_equal(lid, 2 * olid)
        np.testing.assert_array_equal(rid, 2 * orid)


def _device_count():
    import torch
    return torch.cuda.device_count()


@pytest.mark.parametrize("n_dev", [1, 2, 4, 8])
def test_multi_device_text_matches_single_device(n_dev):
    if n_dev > 2 and _device_count() < n_dev:
        pytest.skip(f"needs {n_dev} GPUs")
    sd, user, d, od = synth_user_dictionary()
    utf8, off = synth.make_corpus(sd, 5000, seed=78, log_uniform=(1, 200), unk_frac=0.1, space_frac=0.02, user_csv=user,
                                  user_frac=0.05)
    tok_off, toks = od.tokenize_batch(utf8, off, True, n_threads=8)[:2]
    single = vb.Tokenizer.new(d).ignore_space(True)
    single.set_option("chunk_sentences", 0)
    multi = vb.Tokenizer.new(d, devices=shard_devices(n_dev)).ignore_space(True)
    for mode in MODES + ("wakati",):  # modes switch between calls (and back)
        eoff, etext = vo.format_batch(od, utf8, off, tok_off, toks, mode)
        assert_text_equal(single.output_mode(mode).tokenize_batch(utf8=utf8, byte_offsets=off), eoff, etext)
        multi.output_mode(mode)
        for _ in range(2):  # the second call reuses the shards' buffers and the pinned result pool
            res = multi.tokenize_batch(utf8=utf8, byte_offsets=off)
            assert_batch_equal(res, tok_off, toks)
            assert_text_equal(res, eoff, etext)
        # fewer sentences than devices, only empty sentences, the empty batch, empty shards among full ones
        for sents in (["東京都"], ["", "", ""], [], ["a"] * 3 + [""] * 5):
            u8, o = vb.Tokenizer.pack(sents)
            a = single.tokenize_batch(utf8=u8, byte_offsets=o)
            b = multi.tokenize_batch(utf8=u8, byte_offsets=o)
            assert_batch_equal(b, a.tok_offsets, a.tokens)
            assert_text_equal(b, *a.text())
    multi.output_mode(None)
    res = multi.tokenize_batch(utf8=utf8, byte_offsets=off)
    assert_batch_equal(res, tok_off, toks)
    with pytest.raises(vb.VibratoError):
        res.text()
    # the output stage needs full token records, on every device
    with pytest.raises(vb.VibratoError):
        vb.Tokenizer.new(d, devices=shard_devices(n_dev)).output_mode("mecab").compact_tokens(True)
    with pytest.raises(vb.VibratoError):
        vb.Tokenizer.new(d, devices=shard_devices(n_dev)).compact_tokens(True).output_mode("mecab")


def test_tokenize_cli_devices_and_batch_lines(golden, tmp_path):
    exe = os.path.join(ROOT, "vibrato_b200", "bin", "tokenize")
    if not os.path.exists(exe):
        pytest.skip("CLIs not built")
    for k, v in golden["resources"].items():
        (tmp_path / k).write_text(v, encoding="utf-8", newline="")
    lines = ["京都東京都京都", "東京 都", "", "kampersanda", "東京県に行く", "", ""] * 3
    text = ("\n".join(lines) + "\n").encode()
    flag_sets = [["--devices", "0", "--batch-lines", "2"], ["--batch-lines", "1"], ["--batch-lines", "1000000"]]
    flag_sets += [["--devices", shard_devices_arg(2)], ["--devices", shard_devices_arg(2), "--batch-lines", "3"]]
    for mode in MODES:
        for where in ("device", "host"):
            base = [exe, "-i", str(tmp_path), "-u", str(tmp_path / "user.csv"), "-O", mode, "-S", "-M", "24", "--format-on", where]
            ref = subprocess.run(base, input=text, capture_output=True, timeout=120)
            assert ref.returncode == 0, ref.stderr.decode()
            assert ref.stdout.count(b"\n") >= len(lines)
            for flags in flag_sets:
                p = subprocess.run(base + flags, input=text, capture_output=True, timeout=120)
                assert p.returncode == 0, p.stderr.decode()
                assert p.stdout == ref.stdout, (mode, where, flags)
    p = subprocess.run([exe, "-i", str(tmp_path), "--batch-lines", "0"], input=text, capture_output=True, timeout=120)
    assert p.returncode == 2
