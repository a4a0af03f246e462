"""Required token boundaries on the GPU (vbt_tokenize_batch_bounded / vbt_tokenize_batch_device_bounded): tokens
bit-identical to the bounded oracle (tests/bounded_oracle.py) on every route — whole batch, the chunked host pipeline,
"small_batch", device-resident input and a multi-device tokenizer (host and device-resident input) —
plus the output text, connection id counts, the input errors and `tokenize --boundary-marker`."""
import os
import subprocess

import numpy as np
import pytest

import adversarial as adv
import vibrato_b200 as vb
from bounded_oracle import BoundedOracle
from oracle import vibrato_oracle as vo
from test_gpu_marginals import shard_devices, shard_devices_arg

pytestmark = pytest.mark.gpu
ROUTES = ("whole", "chunked", "small", "device", "multi", "multi_device")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK_COPIES = 2100  # "chunked": batches are repeated to at least this many sentences, so that the pipeline cuts them
# into several chunks (its first chunk holds 1024 sentences)


def lead_bytes(b):
    return [i for i in range(len(b) + 1) if i == len(b) or (b[i] & 0xC0) != 0x80]


def make_bounds(sents, seed):
    """Per sentence: random lead-byte boundaries (some duplicated, some 0 / len), every 4th sentence none, every 7th
    a boundary at every character."""
    rng = np.random.default_rng(seed)
    out = []
    for i, s in enumerate(sents):
        lb = lead_bytes(s.encode())
        if i % 4 == 3:
            out.append([])
        elif i % 7 == 6:
            out.append(lb)
        else:
            k = int(rng.integers(1, 5))
            v = sorted(int(x) for x in rng.choice(lb, size=min(k, len(lb))))
            out.append(v)
    return out


def d2h(ptr, n, dtype):
    from cuda.bindings import runtime as cudart
    host = np.empty(n, dtype=dtype)
    if n:
        (err,) = cudart.cudaMemcpy(host.ctypes.data, ptr, host.nbytes, cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost)
        assert int(err) == 0
    return host


def make_tokenizer(d, route, ignore_space=False, mgl=0):
    if route.startswith("multi"):
        tok = vb.Tokenizer.new(d, devices=shard_devices(2))
    else:
        tok = vb.Tokenizer.new(d)
    tok.ignore_space(ignore_space).max_grouping_len(mgl)
    if route == "chunked":
        tok.set_option("chunk_sentences", 64)
    if route == "small":
        tok.small_batch(65536)
    return tok


def run(tok, route, sents, bounds):
    """(tok_off, tokens) of a bounded call on `route`."""
    utf8, off = adv.pack(sents)
    if route in ("device", "multi_device"):
        import torch
        bo, bnd = vb.Tokenizer.pack_bounds(bounds)
        d_utf8 = torch.from_numpy(utf8.copy()).cuda()
        d_off = torch.from_numpy(off.astype(np.int64)).cuda()
        d_bo = torch.from_numpy(bo.astype(np.int64)).cuda()
        d_bnd = torch.from_numpy(bnd.astype(np.int32)).cuda() if len(bnd) else torch.zeros(1, dtype=torch.int32).cuda()
        torch.cuda.synchronize()
        a, b, n = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), len(sents), len(utf8),
                                            d_bnd_offsets=d_bo.data_ptr(), d_bnd=d_bnd.data_ptr(), n_bnd=len(bnd))
        return d2h(a, len(sents) + 1, np.uint64), d2h(b, n, vb.TOKEN_DTYPE)
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds)
    if route == "small" and len(utf8) <= 16384:
        assert tok.describe()["last_viterbi"] == "k_small_batch"
    return res.tok_offsets.copy(), res.tokens.copy()


def check(tok, route, bo, sents, bounds):
    e_off, e_toks = bo.tokenize_batch([s.encode() for s in sents], bounds)
    if route == "chunked":  # the same batch repeated: the oracle's result repeats too
        k = -(-CHUNK_COPIES // max(1, len(sents)))
        sents, bounds = sents * k, bounds * k
        per = np.diff(e_off.astype(np.int64))
        e_off = np.zeros(len(sents) + 1, dtype=np.uint64)
        e_off[1:] = np.cumsum(np.tile(per, k))
        e_toks = np.tile(e_toks, k)
    off, toks = run(tok, route, sents, bounds)
    np.testing.assert_array_equal(off, e_off)
    for name in vb.TOKEN_DTYPE.names:
        np.testing.assert_array_equal(toks[name], e_toks[name], err_msg=name)


def golden_dicts(golden, user):
    r = golden["resources"]
    d = vb.SystemDictionaryBuilder.from_readers(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
    od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
    if user:
        d.reset_user_lexicon_from_reader(r["user.csv"])
        od.set_user_csv(r["user.csv"])
    return d, od, r


@pytest.mark.parametrize("route", ROUTES)
def test_golden_fixture(golden, route):
    # (the fixture's unk.def has no KATAKANA entry, so a katakana run keeps a path only where lexicon words cover it:
    # アイアイウ is split after アイ, never inside アイウ)
    sents = [c["input"] for c in golden["tokenizer_cases"]] + ["京都東京都京都", "abcdefgh", "東京   都"]
    for user in (False, True):
        d, od, r = golden_dicts(golden, user)
        for isp, mgl in ((False, 0), (True, 0), (False, 3)):
            tok = make_tokenizer(d, route, isp, mgl)
            bo = BoundedOracle(od, r["char.def"], r["unk.def"], isp, mgl)
            check(tok, route, bo, sents, make_bounds(sents, 1))
            check(tok, route, bo, ["京都東京都京都", "アイアイウ"], [[12], [6]])
            check(tok, route, bo, sents, [[] for _ in sents])


@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("ignore_space", [False, True])
@pytest.mark.parametrize("dictionary", list(adv.FAMILIES) + ["raw", "dual"])
def test_adversarial(dictionary, ignore_space, route):
    if dictionary in adv.FAMILIES:
        d, connector = adv.make_dictionary(dictionary), "matrix"
    else:
        d, connector = adv.make_dictionary("wrap", dual=dictionary == "dual"), dictionary
    if connector == "matrix":
        dev = vb.SystemDictionaryBuilder.from_readers(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    else:
        right, left, cost = d.matrix
        dev = vb.SystemDictionaryBuilder.from_readers_with_bigram_info(d.lex_csv, right, left, cost, d.char_def, d.unk_def,
                                                                       dual_connector=connector == "dual")
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def, dual_connector=connector == "dual")
    dev.reset_user_lexicon_from_reader(d.user_csv)
    od.set_user_csv(d.user_csv)
    n = 200 if route == "chunked" else 60
    sents = adv.make_sentences(d, n, seed=5, max_len=80) + [" ", "a  ", "あ ア  ", "", " a"]
    tok = make_tokenizer(dev, route, ignore_space)
    bo = BoundedOracle(od, d.char_def, d.unk_def, ignore_space)
    check(tok, route, bo, sents, make_bounds(sents, 2))


@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("mgl", [0, 1, 24])
def test_max_grouping_len_and_compact(route, mgl):
    d = adv.make_dictionary("ties", seed=3)
    dev = vb.SystemDictionaryBuilder.from_readers(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    dev.reset_user_lexicon_from_reader(d.user_csv)
    od.set_user_csv(d.user_csv)
    sents = adv.make_sentences(d, 40, seed=11, max_len=120) + ["a" * 40 + "ア" * 30, "1" * 50, "漢" * 30 + " " * 3]
    bounds = make_bounds(sents, 3)
    bo = BoundedOracle(od, d.char_def, d.unk_def, True, mgl)
    tok = make_tokenizer(dev, route, True, mgl)
    check(tok, route, bo, sents, bounds)
    if route not in ("device", "multi_device"):
        tok.compact_tokens(True)
        utf8, off = adv.pack(sents)
        res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds)
        e_off, e_toks = bo.tokenize_batch([s.encode() for s in sents], bounds)
        np.testing.assert_array_equal(res.tok_offsets, e_off)
        for name in vb.TOKEN_DTYPE.names:
            np.testing.assert_array_equal(res.tokens[name], e_toks[name], err_msg=name)


@pytest.mark.parametrize("route", ["whole", "small"])
def test_long_sentence_and_extreme_costs(route):
    """A sentence of more than 16 000 characters (the unpruned k_viterbi2 twin) and the extreme-cost family."""
    d = adv.make_dictionary("extreme")
    dev = vb.SystemDictionaryBuilder.from_readers(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    sents = adv.make_sentences(d, 30, seed=9, max_len=200)
    if route == "whole":
        sents.append("".join(adv.make_sentences(d, 400, seed=4, max_len=80))[:17000])
    tok = make_tokenizer(dev, route)
    check(tok, route, BoundedOracle(od, d.char_def, d.unk_def), sents, make_bounds(sents, 4))


@pytest.mark.parametrize("route", ["whole", "chunked", "small", "multi"])
def test_output_text_and_connid_counts(golden, route):
    d = adv.make_dictionary("ties", seed=2)
    dev = vb.SystemDictionaryBuilder.from_readers(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    sents = adv.make_sentences(d, 200, seed=8, max_len=60) * (11 if route == "chunked" else 1)
    bounds = make_bounds(sents, 5)
    bo = BoundedOracle(od, d.char_def, d.unk_def)
    utf8, off = adv.pack(sents)
    e_off, e_toks = bo.tokenize_batch([s.encode() for s in sents], bounds)
    tok = make_tokenizer(dev, route)
    for mode in ("mecab", "wakati", "detail"):
        tok.output_mode(mode)
        res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds)
        toff, text = res.text()
        x_off, x_text = vo.format_batch(od, utf8, off, e_off, e_toks.astype(vb.TOKEN_DTYPE), mode)
        np.testing.assert_array_equal(toff, x_off)
        assert text == x_text
    tok.output_format("%m\t%pS|%ps-%pe\n", eos="EOS %L\n")
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds)
    # the same format over the oracle's bounded tokens, rendered here: surface, skipped spaces, byte range
    lines = []
    b = utf8.tobytes()
    for i in range(len(sents)):
        s0 = int(off[i])
        prev_end = 0
        for t in e_toks[int(e_off[i]):int(e_off[i + 1])]:
            surf = b[s0 + t["start_byte"]:s0 + t["end_byte"]]
            sp = b[s0 + prev_end:s0 + t["start_byte"]]
            lines.append(surf + b"\t" + sp + b"|" + f"{t['start_byte']}-{t['end_byte']}\n".encode())
            prev_end = int(t["end_byte"])
        lines.append(f"EOS {int(off[i + 1] - off[i])}\n".encode())
    assert res.text()[1] == b"".join(lines)
    # connid_counting counts the constrained lattices, on one device or several
    tok.output_mode(None)
    tok.init_connid_counter()
    tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds)
    lid, rid = tok.connid_counts()
    e_lid, e_rid = bo.connid_counts([s.encode() for s in sents], bounds)
    np.testing.assert_array_equal(np.asarray(lid, dtype=np.uint64), e_lid)
    np.testing.assert_array_equal(np.asarray(rid, dtype=np.uint64), e_rid)


@pytest.mark.parametrize("route", ROUTES)
def test_invalid_boundaries(golden, route):
    d, od, r = golden_dicts(golden, False)
    tok = make_tokenizer(d, route)
    sents = ["東京都に行く", "京都", "abc"]
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    if route == "chunked":
        sents = sents * 800  # several chunks; the bad list sits in the last one
    good = [[6], [], [1, 2]] * (len(sents) // 3)
    # unsorted; past the end; inside 都 (bytes 6-8); past the end of 京都; past the end of "abc"
    bad_lists = ([[9, 6], [], []], [[19], [], []], [[7], [], []], [[], [7], []], [[], [], [4]])
    for bad in bad_lists:
        bnd = good[:-3] + bad
        with pytest.raises(vb.VibratoError) as ei:
            run(tok, route, sents, bnd)
        assert ei.value.kind == "InvalidArgument", bad
        check(tok, route, bo, sents, good)  # the tokenizer is still usable
    # UTF-8 errors keep their code and precede boundary errors
    if route not in ("device", "multi_device"):
        utf8, off = adv.pack(sents)
        broken = utf8.copy()
        broken[1] = 0xFF
        with pytest.raises(vb.VibratoError) as ei:
            tok.tokenize_batch(utf8=broken, byte_offsets=off, boundaries=[[7]] + [[] for _ in sents[1:]])
        assert ei.value.kind == "Utf8"
    check(tok, route, bo, sents, good)


@pytest.mark.parametrize("route", ["whole", "small", "device"])
def test_empty_lists_take_the_unbounded_kernels(golden, route):
    """A bounded call whose lists are all empty launches what the unbounded call launches (no k_mark_bounds, the
    unbounded k_candidates); one boundary adds the marking kernel on the multi-kernel routes."""
    d, od, r = golden_dicts(golden, False)
    tok = make_tokenizer(d, route)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    sents = [c["input"] for c in golden["tokenizer_cases"]]
    utf8, off = adv.pack(sents)
    if route == "device":
        import torch
        d_utf8 = torch.from_numpy(utf8.copy()).cuda()
        d_off = torch.from_numpy(off.astype(np.int64)).cuda()
        tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), len(sents), len(utf8))
    else:
        tok.tokenize_batch(utf8=utf8, byte_offsets=off)
    plain = tok.last_launch_count()
    check(tok, route, bo, sents, [[] for _ in sents])
    assert tok.last_launch_count() == plain
    check(tok, route, bo, sents, [[0, len(s.encode())] if i == 0 else [] for i, s in enumerate(sents)])
    assert tok.last_launch_count() == plain + (0 if route == "small" else 1)


def test_counting_refuses_bounded_calls(golden):
    d, od, r = golden_dicts(golden, False)
    tok = vb.Tokenizer.new(d)
    tok.set_counting(True)
    with pytest.raises(vb.VibratoError) as ei:
        tok.tokenize_batch(["東京都"], boundaries=[[6]])
    assert ei.value.kind == "InvalidArgument"
    tok.set_counting(False)
    res = tok.tokenize_batch(["東京都"], boundaries=[[6]])
    assert [res.sentence_tokens(0)[i].surface() for i in range(res.num_tokens(0))] == ["東京", "都"]


def test_worker_reset_sentence_with_boundaries(golden):
    d, od, r = golden_dicts(golden, False)
    w = vb.Tokenizer.new(d).new_worker()
    w.reset_sentence("京都東京都京都", boundaries=[12])
    w.tokenize()
    assert [t.surface() for t in w.token_iter()] == ["京都", "東京", "都", "京都"]
    w.reset_sentence("京都東京都京都")
    w.tokenize()
    assert "東京都" in [t.surface() for t in w.token_iter()]


def test_tokenize_cli_boundary_marker(golden, tmp_path):
    """`tokenize --boundary-marker '|'`: the same bytes with every batching (whole input, --batch-lines, one line at a
    time on a terminal, a two-entry --devices) and each output mode, equal to the bounded tokens of the API."""
    from test_gpu_small_batch import _run_on_pty
    exe = os.path.join(ROOT, "vibrato_b200", "bin", "tokenize")
    if not os.path.exists(exe):
        pytest.skip("CLIs not built")
    r = golden["resources"]
    for k, v in r.items():
        (tmp_path / k).write_text(v, encoding="utf-8", newline="")
    lines = ["京都|東京都京都", "|東京 | 都|", "", "kamper||sanda", "東京県に行く", "|", "abc|def"] * 3
    text = ("\n".join(lines) + "\n").encode()
    plain = [ln.replace("|", "") for ln in lines]
    bnds = []
    for ln in lines:
        b, w = [], 0
        for ch in ln:
            if ch == "|":
                if not b or b[-1] != w:
                    b.append(w)
            else:
                w += len(ch.encode())
        bnds.append(b)
    d, _, _ = golden_dicts(golden, False)
    for mode in ("mecab", "wakati", "detail"):
        expect = vb.Tokenizer.new(d).output_mode(mode).tokenize_batch(plain, boundaries=bnds).text()[1]
        for where in ("device", "host"):
            base = [exe, "-i", str(tmp_path), "-O", mode, "--format-on", where, "--boundary-marker", "|"]
            ref = subprocess.run(base, input=text, capture_output=True, timeout=120)
            assert ref.returncode == 0, ref.stderr.decode()
            assert ref.stdout == expect, (mode, where)
            runs = [base + ["--batch-lines", "2"]] + [base + ["--devices", shard_devices_arg(2)]]
            for cmd in runs:
                out = subprocess.run(cmd, input=text, capture_output=True, timeout=120)
                assert out.returncode == 0, out.stderr.decode()
                assert out.stdout == ref.stdout, (mode, where, cmd[-2:])
            assert _run_on_pty(base, text) == ref.stdout, (mode, where)
    fmt = [exe, "-i", str(tmp_path), "-F", "%m[%ps]\\n", "--eos-format", "%S\\n", "--boundary-marker", "|"]
    out = subprocess.run(fmt, input="東京|都\n".encode(), capture_output=True, timeout=120)
    assert out.returncode == 0, out.stderr.decode()
    assert out.stdout.decode() == "東京[0]\n都[6]\n東京都\n"
    bad = subprocess.run(base[:-1] + ["||"], input=text, capture_output=True, timeout=120)
    assert bad.returncode == 2
