"""The single-pass front (count_chars + slot-offset scan + decode) and back (path walk + token-offset scan + records)
kernels at their edges, against the oracle: sentence counts around the tile sizes (32 and 256), empty batches and
sentences, text larger than a tile's staging buffer, input errors in the last tile only, the slot-overflow re-run, chunk
boundaries of the host pipeline and 16-byte records."""
import numpy as np
import pytest

import vibrato_b200 as vb
from test_gpu_parity import dicts

pytestmark = pytest.mark.gpu
ROUTES = ("whole", "chunked", "compact", "device")


def base_sents(golden):
    return [c["input"] for c in golden["tokenizer_cases"]] + ["東京に行った。", "", "X" * 40, "京都"]


def make(d, route):
    tok = vb.Tokenizer.new(d)
    if route == "chunked":
        tok.set_option("chunk_sentences", 64)
    if route == "compact":
        tok.compact_tokens(True)
    return tok


def run(tok, route, utf8, off):
    if route != "device":
        res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
        return res.tok_offsets, res.tokens
    import torch
    from cuda.bindings import runtime as cudart
    n_sent = len(off) - 1
    d_utf8 = torch.from_numpy(utf8.copy() if len(utf8) else np.zeros(1, np.uint8)).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    torch.cuda.synchronize()
    a, b, n = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), n_sent, len(utf8))
    tok_off = np.empty(n_sent + 1, dtype=np.uint64)
    toks = np.empty(n, dtype=vb.TOKEN_DTYPE)
    (err,) = cudart.cudaMemcpy(tok_off.ctypes.data, a, tok_off.nbytes, cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost)
    assert int(err) == 0
    if n:
        (err,) = cudart.cudaMemcpy(toks.ctypes.data, b, toks.nbytes, cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost)
        assert int(err) == 0
    return tok_off, toks


def check(d, od, sents, route, tok=None):
    utf8, off = vb.Tokenizer.pack(sents)
    tok = tok or make(d, route)
    tok_off, toks = run(tok, route, utf8, off)
    exp_off, exp, _ = od.tokenize_batch(utf8, off)
    np.testing.assert_array_equal(np.asarray(tok_off, dtype=np.uint64), np.asarray(exp_off, dtype=np.uint64))
    for name in vb.TOKEN_DTYPE.names:
        np.testing.assert_array_equal(toks[name], exp[name], err_msg=name)


@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 1000])
def test_counts_around_tiles(golden, route, n):
    d, od = dicts(golden, True)
    pool = base_sents(golden)
    check(d, od, [pool[(i * 7) % len(pool)] for i in range(n)], route)


@pytest.mark.parametrize("route", ("whole", "chunked", "device"))
def test_empty_batch_and_sentences(golden, route):
    d, od = dicts(golden)
    tok = make(d, route)
    check(d, od, [], route, tok)
    check(d, od, [""], route, tok)
    check(d, od, [""] * 70, route, tok)
    check(d, od, ["", "東京都", ""] * 40, route, tok)


@pytest.mark.parametrize("route", ROUTES)
def test_text_past_the_staging_buffer(golden, route):
    d, od = dicts(golden, True)
    pool = base_sents(golden)
    sents = [pool[i % len(pool)] for i in range(100)]
    sents[40] = "東京都に" * 1500   # 18 000 bytes: its tile reads global memory
    sents[70] = "X" * 300 + "9" * 300  # 600 characters in a staged tile: more than a warp decodes in shared memory
    sents[99] = "京都" * 300
    check(d, od, sents, route)


@pytest.mark.parametrize("route", ("whole", "device"))
def test_input_errors_in_the_last_tile(golden, route):
    d, _ = dicts(golden)
    pool = base_sents(golden)
    sents = [pool[i % len(pool)] for i in range(300)]
    utf8, off = vb.Tokenizer.pack(sents)
    bad = utf8.copy()
    bad[int(off[-2])] = 0xFF  # the last sentence starts with a byte that UTF-8 never has
    tok = make(d, route)
    with pytest.raises(Exception):
        run(tok, route, bad, off)
    off2 = off.copy()
    off2[-2] = off2[-3] - 1  # the last but one sentence ends before it starts
    with pytest.raises(Exception):
        run(tok, route, utf8, off2)
    # the tokenizer stays usable
    d2, od = dicts(golden)
    check(d2, od, sents, route, tok)


@pytest.mark.parametrize("route", ROUTES)
def test_slot_overflow_rerun(golden, route):
    d, od = dicts(golden)
    tok = make(d, route)
    tok.set_option("chars_estimate_permille", 1)  # the first batch underestimates characters per byte
    check(d, od, ["X" * 50, "9" * 30, "東京都"] * 200, route, tok)


def test_chunk_boundaries(golden):
    d, od = dicts(golden, True)
    pool = base_sents(golden)
    for n in (63, 64, 65, 129, 300):
        check(d, od, [pool[(i * 5) % len(pool)] for i in range(n)], "chunked")


@pytest.mark.parametrize("route", ("whole", "compact", "device"))
@pytest.mark.parametrize("n", [40000, 40001, 40255])
def test_large_back_tiles(golden, route, n):
    # enough sentences for the 256-sentence back tiles on any H100 (132 SMs x 256 < 40 000)
    d, od = dicts(golden, True)
    pool = base_sents(golden)
    check(d, od, [pool[(i * 7) % len(pool)] for i in range(n)], route)
