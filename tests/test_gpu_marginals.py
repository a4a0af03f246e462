"""Marginal probabilities on the GPU (vbt_tokenizer_set_marginals): the tokens are unchanged, the probabilities match
the forward-backward restatement (tests/marginal_oracle.py), and they are bit-identical on every route — whole
batch, the chunked host pipeline, compact records, "small_batch" (which steps aside), device-resident input,
bounded calls, every K3 variant and multi-device tokenizers."""
import ctypes as C

import numpy as np
import pytest

import adversarial as adv
import marginal_oracle as mo
import vibrato_b200 as vb
from bounded_oracle import BoundedOracle
from oracle import vibrato_oracle as vo
from vibrato_b200._native import lib

pytestmark = pytest.mark.gpu
ROUTES = ("whole", "chunked", "compact", "small", "device", "viterbi0", "unpruned", "multi", "multi_device")
THETA = 0.01


def n_gpus():
    import torch
    return torch.cuda.device_count()


def shard_devices(n):
    """The devices of an n-entry multi-device tokenizer: n distinct GPUs when the machine has them, else device 0 n
    times (each entry is its own shard engine, so the sharded path runs on one GPU too)."""
    return list(range(n)) if n_gpus() >= n else [0] * n


def shard_devices_arg(n):
    """shard_devices(n) as a `--devices` value."""
    return ",".join(map(str, shard_devices(n)))


def d2h(ptr, n, dtype):
    from cuda.bindings import runtime as cudart
    host = np.empty(n, dtype=dtype)
    if n:
        (err,) = cudart.cudaMemcpy(host.ctypes.data, ptr, host.nbytes, cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost)
        assert int(err) == 0
    return host


def make_tokenizer(d, route, ignore_space=False, mgl=0, theta=THETA):
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
    return tok.marginals(theta)


def run(tok, route, sents, bounds=None):
    """(tok_off, tokens, token_probs, path_probs) of one call on `route`."""
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
        a, b, n = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), len(sents), len(utf8), **kw)
        tp, pp = tok.last_device_marginals()
        return (d2h(a, len(sents) + 1, np.uint64), d2h(b, n, vb.TOKEN_DTYPE), d2h(tp, n, np.float32),
                d2h(pp, len(sents), np.float32))
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, boundaries=bounds)
    if route == "small":
        assert tok.describe()["last_viterbi"] != "k_small_batch"
    res.close()
    return res.tok_offsets, res.tokens, res.token_probs, res.path_probs


def check_against(bo, sents, got, theta=THETA, bounds=None):
    off, toks, tp, pp = got
    e_off, e_toks = bo.tokenize_batch([s.encode() for s in sents], bounds)
    np.testing.assert_array_equal(off, e_off)
    for name in vb.TOKEN_DTYPE.names:
        np.testing.assert_array_equal(toks[name], e_toks[name], err_msg=name)
    e_tp, e_pp = mo.batch_marginals(bo, [s.encode() for s in sents], theta, bounds)
    mo.assert_f32_close(tp, e_tp, what="token_probs")
    mo.assert_f32_close(pp, e_pp, what="path_probs")


def golden_dicts(golden, user):
    r = golden["resources"]
    d = vb.SystemDictionaryBuilder.from_readers(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
    od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
    if user:
        d.reset_user_lexicon_from_reader(r["user.csv"])
        od.set_user_csv(r["user.csv"])
    return d, od, r


def adversarial_dicts(family):
    if family in adv.FAMILIES:
        d, connector = adv.make_dictionary(family), "matrix"
    else:
        d, connector = adv.make_dictionary("wrap", dual=family == "dual"), family
    if connector == "matrix":
        dev = vb.SystemDictionaryBuilder.from_readers(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    else:
        right, left, cost = d.matrix
        dev = vb.SystemDictionaryBuilder.from_readers_with_bigram_info(d.lex_csv, right, left, cost, d.char_def,
                                                                       d.unk_def, dual_connector=connector == "dual")
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def, dual_connector=connector == "dual")
    dev.reset_user_lexicon_from_reader(d.user_csv)
    od.set_user_csv(d.user_csv)
    return d, dev, od


def golden_sents(golden):
    return [c["input"] for c in golden["tokenizer_cases"]] + ["京都東京都京都", "abcdefgh", "東京   都", "", "kampersanda"]


def test_tokens_unchanged_and_probabilities_match(golden):
    """Whole batch: the token records are those of marginals off, and the probabilities match the restatement."""
    sents = golden_sents(golden)
    for user in (False, True):
        d, od, r = golden_dicts(golden, user)
        for isp, mgl in ((False, 0), (True, 0), (False, 3)):
            tok = make_tokenizer(d, "whole", isp, mgl)
            bo = BoundedOracle(od, r["char.def"], r["unk.def"], isp, mgl)
            got = run(tok, "whole", sents)
            check_against(bo, sents, got)
            off_plain, toks_plain, _, _ = run(make_tokenizer(d, "whole", isp, mgl, theta=0), "whole", sents)
            np.testing.assert_array_equal(got[0], off_plain)
            np.testing.assert_array_equal(got[1], toks_plain)


@pytest.mark.parametrize("route", ROUTES)
def test_routes_bit_identical(golden, route):
    d, od, r = golden_dicts(golden, True)
    sents = golden_sents(golden) * 40 + [""] * 70 + golden_sents(golden) * 30  # empty runs across chunk edges
    ref = run(make_tokenizer(d, "whole", True), "whole", sents)
    got = run(make_tokenizer(d, route, True), route, sents)
    np.testing.assert_array_equal(got[0], ref[0])
    if route != "compact":
        np.testing.assert_array_equal(got[1], ref[1])
    np.testing.assert_array_equal(got[2], ref[2])
    np.testing.assert_array_equal(got[3], ref[3])


@pytest.mark.parametrize("route", ("whole", "chunked", "device", "multi", "multi_device"))
def test_bounded(golden, route):
    d, od, r = golden_dicts(golden, False)
    sents = ["京都東京都京都", "アイアイウ", "東京   都", ""] * 30
    bounds = [[12], [6], [], []] * 30
    tok = make_tokenizer(d, route, True)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"], True)
    got = run(tok, route, sents, bounds)
    check_against(bo, sents, got, bounds=bounds)
    ref = run(make_tokenizer(d, "whole", True), "whole", sents, bounds)
    for a, b in zip(got[2:], ref[2:]):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("ignore_space", [False, True])
@pytest.mark.parametrize("family", list(adv.FAMILIES) + ["raw", "dual"])
def test_adversarial(family, ignore_space):
    d, dev, od = adversarial_dicts(family)
    sents = adv.make_sentences(d, 60, seed=5, max_len=60) + [" ", "a  ", "あ ア  ", "", " a"]
    theta = THETA if family in adv.FAMILIES else 1e-6  # the wrap family's costs are near +-2^31
    tok = make_tokenizer(dev, "whole", ignore_space, theta=theta)
    bo = BoundedOracle(od, d.char_def, d.unk_def, ignore_space)
    check_against(bo, sents, run(tok, "whole", sents), theta=theta)
    plain = run(make_tokenizer(dev, "whole", ignore_space, theta=0), "whole", sents)
    got = run(tok, "whole", sents)
    np.testing.assert_array_equal(got[1], plain[1])


def test_large_theta_tie_fractions():
    d, dev, od = adversarial_dicts("ties")
    sents = [s for s in adv.make_sentences(d, 80, seed=9, max_len=30) if s]
    tok = make_tokenizer(dev, "whole", theta=60.0)
    _, _, tp, _ = run(tok, "whole", sents)
    bo = BoundedOracle(od, d.char_def, d.unk_def)
    k, seen = 0, 0
    for s in sents:
        lat = mo.Lattice(bo, s.encode())
        frac = mo.tie_fractions(lat)
        for n in lat.best_path():
            assert abs(float(tp[k]) - float(frac[n])) <= 1e-5, (s, frac[n], tp[k])
            seen += 0 < frac[n] < 1
            k += 1
    assert k == len(tp) and seen


def test_long_sentence(golden):
    """A 20 000-character sentence (past kPruneMaxChars) among short ones: finite, and as the restatement says."""
    d, od, r = golden_dicts(golden, False)
    long = ("京都東京都京都" + "abc " + "東京") * 1540
    long = long[:20000]
    sents = ["京都", long, "東京都"]
    tok = make_tokenizer(d, "whole")
    got = run(tok, "whole", sents)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"])
    check_against(bo, sents, got)


def test_empty_batches(golden):
    d, _, _ = golden_dicts(golden, False)
    for route in ("whole", "device"):
        tok = make_tokenizer(d, route)
        off, toks, tp, pp = run(tok, route, [])
        assert len(tp) == 0 and len(pp) == 0
        off, toks, tp, pp = run(tok, route, ["", "", ""])
        assert len(tp) == 0 and list(pp) == [1.0, 1.0, 1.0]


def test_refusals(golden):
    d, _, _ = golden_dicts(golden, False)
    tok = vb.Tokenizer.new(d)
    for bad in (-1.0, float("nan"), float("inf")):
        with pytest.raises(vb.VibratoError) as e:
            tok.marginals(bad)
        assert e.value.kind == "InvalidArgument"
    res = tok.tokenize_batch(["京都"])
    assert res.token_probs is None and res.path_probs is None
    a, b = C.c_void_p(), C.c_void_p()
    assert lib().vbt_result_marginals(res._h, C.byref(a), C.byref(b)) == 1
    with pytest.raises(vb.VibratoError):
        res.sentence_tokens(0)[0].prob()
    import torch
    utf8, off = adv.pack(["京都"])
    d_utf8, d_off = torch.from_numpy(utf8.copy()).cuda(), torch.from_numpy(off.astype(np.int64)).cuda()
    torch.cuda.synchronize()
    tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), 1, len(utf8))
    with pytest.raises(vb.VibratoError):
        tok.last_device_marginals()


def test_counting_hooks_and_rebuild(golden):
    """Counting and connection-id counting (round-1 K3) give the same probabilities; a rebuilt engine keeps them on."""
    d, od, r = golden_dicts(golden, False)
    sents = golden_sents(golden)
    ref = run(make_tokenizer(d, "whole"), "whole", sents)
    tok = make_tokenizer(d, "whole")
    tok.set_counting(True)
    got = run(tok, "whole", sents)
    np.testing.assert_array_equal(got[2], ref[2])
    tok.set_counting(False)
    tok.init_connid_counter()
    np.testing.assert_array_equal(run(tok, "whole", sents)[2], ref[2])
    tok = make_tokenizer(d, "whole")
    tok.max_grouping_len(0)  # rebuilds the engine: the setting is replayed
    np.testing.assert_array_equal(run(tok, "whole", sents)[2], ref[2])


def test_launch_count_stages_and_worker(golden):
    d, _, _ = golden_dicts(golden, False)
    sents = golden_sents(golden)
    tok = vb.Tokenizer.new(d)
    tok.tokenize_batch(sents)
    n_off, stages = tok.last_launch_count(), list(tok.last_stage_ms())
    tok.marginals(THETA)
    res = tok.tokenize_batch(sents)
    assert tok.last_launch_count() == n_off + 2 and list(tok.last_stage_ms()) == stages
    w = tok.new_worker()
    w.reset_sentence("京都東京都京都")
    w.tokenize()
    probs = [t.prob() for t in w.token_iter()]
    i = sents.index("京都東京都京都")
    a, b = int(res.tok_offsets[i]), int(res.tok_offsets[i + 1])
    assert probs == [float(x) for x in res.token_probs[a:b]]
    assert [t.prob() for t in res.sentence_tokens(i)] == probs
    tok.marginals(None)
    assert tok.tokenize_batch(sents).token_probs is None


def test_report_worst_error():
    """Prints the largest float32 ulp distance from the reference that the tests of this session have seen (those
    above, and those of every test file that ran before it)."""
    print(f"marginals: worst distance from the reference = {mo.F32_ULPS['worst']} float32 ulps")


def parse_pp(text, sents):
    """The %pP values of a '%m\\t%pP\\n' text, per sentence in order."""
    vals = []
    for line in text.decode().split("\n"):
        if line and line != "EOS":
            vals.append(float(line.rsplit("\t", 1)[1]))
    return np.array(vals, dtype=np.float64)


@pytest.mark.parametrize("route", ("whole", "chunked", "multi"))
def test_pP_format(golden, route):
    """%pP prints round(p * 1e6) as d.dddddd, on the host routes that format on the device."""
    d, od, r = golden_dicts(golden, True)
    sents = golden_sents(golden) * (30 if route == "chunked" else 1)
    tok = make_tokenizer(d, route, True).output_format("%m\t%pP\n", eos="EOS\n")
    res = tok.tokenize_batch(sents)
    _, text = res.text()
    got = parse_pp(text, sents)
    for line in text.decode().split("\n"):
        if line and line != "EOS":
            v = line.rsplit("\t", 1)[1]
            assert len(v) == 8 and v[1] == "." and v[0] in "01"
    np.testing.assert_array_equal(got, np.round(res.token_probs.astype(np.float64) * 1e6) / 1e6)
    bo = BoundedOracle(od, r["char.def"], r["unk.def"], True)
    exp, _ = mo.batch_marginals(bo, [s.encode() for s in sents], THETA)
    exp = np.asarray(exp)
    # the printed micro-units are the rounding of a value within two float32 steps (2^-22 relative) of the reference
    assert got.shape == exp.shape and np.all(np.abs(np.rint(got * 1e6) - exp * 1e6) <= 0.5 + 2.4e-7 * exp * 1e6)


def test_pP_refusals(golden):
    d, _, _ = golden_dicts(golden, False)
    tok = vb.Tokenizer.new(d)
    with pytest.raises(vb.VibratoError) as e:  # no value without marginals, as before
        tok.output_format("%m\t%pP\n")
    assert "%pP" in str(e.value)
    tok.marginals(THETA).output_format("%m\t%pP\n")
    with pytest.raises(vb.VibratoError) as e:
        tok.marginals(0)
    assert "format" in str(e.value)
    assert tok.tokenize_batch(["京都"]).token_probs is not None  # still on
    tok.output_format("%m\n").marginals(0)  # a format without %pP: marginals may go
    assert tok.tokenize_batch(["京都"]).token_probs is None
    for pa in ("%pA", "%pB"):
        with pytest.raises(vb.VibratoError):
            tok.marginals(THETA).output_format(pa)


def test_tokenize_cli_marginal(golden, tmp_path):
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
    d, _, _ = golden_dicts(golden, True)
    tok = vb.Tokenizer.new(d).ignore_space(True).marginals(THETA).output_format("%m\t%pP\n")
    _, want = tok.tokenize_batch(plain, boundaries=[[len(s[:s.index("|")].encode())] if "|" in s else [] for s in lines]).text()
    base = [exe, "-i", str(tmp_path), "-u", str(tmp_path / "user.csv"), "-S"]
    for flags in ([], ["--batch-lines", "1"]):
        p = subprocess.run(base + ["-m", "-t", str(THETA), "-F", "%m\t%pP\n", "--boundary-marker", "|"] + flags,
                           input=data, capture_output=True, timeout=120)
        assert p.returncode == 0, p.stderr.decode()
        assert p.stdout == want
    mecab = subprocess.run(base + ["-O", "mecab"], input=data, capture_output=True, timeout=120)
    p = subprocess.run(base + ["-m", "--theta", str(THETA), "-O", "mecab"], input=data, capture_output=True, timeout=120)
    assert p.returncode == 0 and p.stdout == mecab.stdout  # -O output is unchanged
    for bad in (["-m"], ["-t", "0.5"], ["-m", "-t", "x"]):
        assert subprocess.run(base + bad, input=data, capture_output=True, timeout=120).returncode == 2
    p = subprocess.run(base + ["-m", "-t", "-1"], input=data, capture_output=True, timeout=120)
    assert p.returncode == 1 and b"theta" in p.stderr
