"""The multi-device shard path (multi_engine.cu) against the single-device whole-batch call, which the other suites pin
to the oracles: every output array and every text, every shape of cut the byte split makes, bounded and span calls,
the device-resident gather, the input errors and their precedence across shards, the counters, the Worker and the
`tokenize --devices` CLI.  shard_devices(n) repeats device 0 when the machine has fewer than n GPUs, so all of it
runs on one GPU (each entry is its own shard engine); the NCCL transport, cross-device peer copies and pinning
shard threads to different NUMA nodes need distinct devices and are not reached that way."""
import os
import subprocess

import numpy as np
import pytest

import adversarial as adv
import vibrato_b200 as vb
from span_oracle import SpanOracle
from test_gpu_marginals import golden_dicts, golden_sents, shard_devices
from test_gpu_spans import make_spans

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = (2, 3, 5)
THETA = 0.01
N_SAMP = 3
LONG = "京都東京都京都" * 2300  # 16 100 characters: beyond the pruned k_viterbi2's limit, so its shard takes the twin
ARRAYS = ("tok_offsets", "tokens", "compact", "token_probs", "path_probs", "entropies", "log_path_probs",
          "boundary_offsets", "boundary_probs", "node_offsets", "nodes", "node_links", "node_probs", "node_margins",
          "sample_offsets", "samples", "posterior_offsets", "posterior_tokens", "posterior_probs", "posterior_gains")
FORMAT = ("%m\t%f[0]\t%c\n", "%m\t?%pP\n", "BOS\n", "EOS\n")


# ---- option sets: each configures a tokenizer from scratch or from any other set --------------------------------------

def reset(tok):
    """Every output option off, in an order each step accepts."""
    tok.output_mode(None).posterior(None).sampling(0).uncertainty(False).lattice(False).marginals(None)
    return tok.compact_tokens(False).sample_base(0)


OPTIONS = {
    "tokens": lambda t: t,
    "compact": lambda t: t.compact_tokens(True),
    "marginals": lambda t: t.marginals(THETA),
    "uncertainty": lambda t: t.marginals(THETA).uncertainty(boundary_probs=True),
    "lattice": lambda t: t.marginals(THETA).lattice(True),
    "margin0": lambda t: t.lattice(True, margin=0),
    "margin": lambda t: t.marginals(THETA).lattice(True, margin=2000),
    "samples": lambda t: t.sampling(N_SAMP, THETA, 7).sample_base(11),
    "samples_seed2": lambda t: t.sampling(2, THETA, 2 ** 63 + 5).sample_base(3),
    "posterior": lambda t: t.marginals(THETA).posterior(1.0),
    "all": lambda t: t.marginals(THETA).uncertainty(boundary_probs=True).lattice(True, margin=500)
                      .sampling(N_SAMP, THETA, 9).sample_base(1).posterior(2.0),
}
TEXT_OPTIONS = {  # host results only: the device-resident route makes no text
    "mecab": lambda t: t.output_mode("mecab"),
    "wakati": lambda t: t.output_mode("wakati"),
    "detail": lambda t: t.output_mode("detail"),
    "format": lambda t: t.marginals(THETA).output_format(*FORMAT),
    "lattice_text": lambda t: t.marginals(THETA).lattice(True, text=True).output_mode("mecab"),
    "sample_text": lambda t: t.sampling(N_SAMP, THETA, 5, text=True).sample_base(2).output_mode("wakati"),
    "posterior_text": lambda t: t.marginals(THETA).posterior(1.0, text=True).output_mode("mecab"),
    "all_text": lambda t: OPTIONS["all"](t).output_mode("mecab"),
}


def configured(tok, name):
    return {**OPTIONS, **TEXT_OPTIONS}[name](reset(tok))


# ---- the batch shapes ---------------------------------------------------------------------------------------------------

def cuts(off, n):
    """multi_engine.cu split_by_bytes: the first sentence of each of the n shards, and len(off) - 1 at the end."""
    n_sent = len(off) - 1
    cut = [0] + [n_sent] * n
    first = int(off[0]) if n_sent else 0
    total = int(off[-1]) - first if n_sent else 0
    for i in range(1, n):
        target = first + total // n * i
        cut[i] = max(cut[i - 1], min(int(np.searchsorted(off, target, side="left")), n_sent))
    return cut


def shapes(golden):
    base = golden_sents(golden)
    return {
        "mixed": base * 6 + [""] * 9 + base * 4,
        "fewer": ["東京都", "京都"],  # fewer sentences than entries (for 3 and 5)
        "one": ["京都東京都京都"],  # the trailing shards are empty; the last delivers every closing offset
        "only_empty": [""] * 4,  # every cut is 0: the last shard takes all
        "empty_batch": [],
        "gaps": ["ab", "東京都" * 400, "cd", "ef", "京都"],  # several cuts coincide: empty shards between full ones
        "long_first": [LONG] + base * 3,  # only the first shard holds a sentence beyond the pruned kernel's limit
    }


def pack(sents, prefix=0, pinned=False):
    """(utf8, byte_offsets) of the sentences after `prefix` unrelated bytes (byte_offsets[0] = prefix), in pageable
    or pinned host memory (a pinned torch tensor's numpy view)."""
    utf8, off = adv.pack(sents)
    utf8 = np.concatenate([np.frombuffer(b"x" * prefix, np.uint8), utf8])
    off = off + np.uint64(prefix)
    if pinned:
        import torch
        pu = torch.empty(max(1, len(utf8)), dtype=torch.uint8, pin_memory=True).numpy()[:len(utf8)]
        po = torch.empty(len(off), dtype=torch.int64, pin_memory=True).numpy().view(np.uint64)
        pu[:], po[:] = utf8, off
        utf8, off = pu, po
    return utf8, off


# ---- one call, every array as bytes ------------------------------------------------------------------------------------

def host_call(tok, utf8, off, **kw):
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off, **kw)
    got = {name: getattr(res, name).tobytes() for name in ARRAYS if getattr(res, name) is not None}
    try:
        o, t = res.text()
        got["text"] = (o.tobytes(), t)
    except vb.VibratoError as e:
        got["text"] = str(e)
    res.close()
    return got


def d2b(ptr, nbytes):
    from cuda.bindings import runtime as cudart
    host = np.empty(nbytes, np.uint8)
    if nbytes:
        assert ptr
        (err,) = cudart.cudaMemcpy(host.ctypes.data, ptr, nbytes, cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost)
        assert int(err) == 0
    return host.tobytes()


def to_device(*arrays):
    import torch
    out = [torch.from_numpy(np.array(a) if len(a) else np.zeros(1, a.dtype)).cuda() for a in arrays]
    torch.cuda.synchronize()
    return out


def device_call(tok, utf8, off, n_bytes=None, bounds=None, spans=None):
    """tokenize_batch_device with the input on device 0, then every last_device_* accessor: its arrays as bytes, or
    the refusal's message."""
    n = len(off) - 1
    t = to_device(utf8, off.astype(np.int64))
    kw = {}
    if bounds is not None or spans is not None:
        bo, bnd = vb.Tokenizer.pack_bounds(bounds if bounds is not None else [[] for _ in range(n)])
        tb = to_device(bo.astype(np.int64), bnd.astype(np.int32))
        t += tb
        kw = dict(d_bnd_offsets=tb[0].data_ptr(), d_bnd=tb[1].data_ptr(), n_bnd=len(bnd))
        if spans is not None:
            so, recs, pats = vb.Tokenizer.pack_spans(spans)
            ts = to_device(so.astype(np.int64), recs.astype(np.int32).reshape(-1))
            t += ts
            kw.update(d_span_offsets=ts[0].data_ptr(), d_spans=ts[1].data_ptr(), n_spans=len(recs), patterns=pats)
    a, b, nt = tok.tokenize_batch_device(t[0].data_ptr(), t[1].data_ptr(), n, len(utf8) if n_bytes is None else n_bytes,
                                         **kw)
    rec = 16 if tok._options.get("compact_tokens") else 24
    got = {"tokens": (d2b(a, (n + 1) * 8), d2b(b, nt * rec))}

    def grab(name, f):
        try:
            got[name] = f()
        except vb.VibratoError as e:
            got[name] = str(e)

    def marg():
        tp, pp = tok.last_device_marginals()
        return d2b(tp, nt * 4), d2b(pp, n * 4)

    def unc():
        e, lp, po, pb, npos = tok.last_device_uncertainty()
        return d2b(e, n * 8), d2b(lp, n * 8), d2b(po, (n + 1) * 8) if po else None, d2b(pb, npos * 4)

    def lat():
        no, nodes, links, nprob, nn = tok.last_device_lattice()
        return (d2b(no, (n + 1) * 8), d2b(nodes, nn * 24), d2b(links, nn * vb.LINK_DTYPE.itemsize),
                d2b(nprob, nn * 4) if nprob else None, nn)

    def margins():
        nn = tok.last_device_lattice()[4]
        return d2b(tok.last_device_lattice_margins(), nn * 8)

    def samp():
        so, s, ns = tok.last_device_samples()
        return d2b(so, (n * tok._sampling[0] + 1) * 8), d2b(s, ns * 24)

    def post():
        po, pt, pp, pg, npt = tok.last_device_posterior()
        return d2b(po, (n + 1) * 8), d2b(pt, npt * 24), d2b(pp, npt * 4), d2b(pg, n * 8)

    for name, f in (("marginals", marg), ("uncertainty", unc), ("lattice", lat), ("margins", margins),
                    ("samples", samp), ("posterior", post)):
        grab(name, f)
    return got


def assert_same(got, ref, what):
    assert got.keys() == ref.keys(), what
    for name in ref:
        assert got[name] == ref[name], (what, name)


def error_of(fn):
    with pytest.raises(vb.VibratoError) as e:
        fn()
    return e.value.code, str(e.value)


# ---- outputs ------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def golden_dict(golden):
    return golden_dicts(golden, True)


@pytest.mark.parametrize("n", SIZES)
def test_every_output_and_shape_on_host(golden, golden_dict, n):
    """Host batches: every option set (switched on one sharded tokenizer, so that a pooled result carries other
    arrays than the last one) on every batch shape, from pageable and pinned memory, with byte_offsets[0] > 0; every
    array and the text byte for byte against the single device, twice, and the tokens against the C oracle."""
    d, od, _ = golden_dict
    multi = vb.Tokenizer.new(d, devices=shard_devices(n))
    info = multi.describe()
    assert info["devices"] == shard_devices(n)
    if len(set(shard_devices(n))) < n:
        assert info["dictionary_transport"] == "cudaMemcpyPeer" and info["token_gather"] == "cudaMemcpyPeer"
    single = vb.Tokenizer.new(d)
    sh = shapes(golden)
    # the shapes do what their names say
    _, o = adv.pack(sh["one"])
    assert cuts(o, n) == [0] + [1] * n
    _, o = adv.pack(sh["only_empty"])
    assert cuts(o, n) == [0] * n + [4]
    _, o = adv.pack(sh["gaps"])
    c = cuts(o, n)
    assert c[1] == 2 and (n == 2 or c[2] == 2)  # with 3 or more entries the second shard is empty
    _, o = adv.pack(sh["long_first"])
    assert cuts(o, n)[1] == 1
    for opt in list(OPTIONS) + list(TEXT_OPTIONS):
        configured(multi, opt)
        configured(single, opt)
        for shape, sents in sh.items():
            e_off, e_toks, _ = od.tokenize_batch(*adv.pack(sents))
            for prefix, pinned in ((0, False), (5, True)) if shape in ("mixed", "gaps", "one") else ((0, False),):
                utf8, off = pack(sents, prefix, pinned)
                ref = host_call(single, utf8, off)
                if opt == "tokens":
                    assert ref["tok_offsets"] == e_off.tobytes() and ref["tokens"] == e_toks.tobytes()
                for _ in range(2):
                    got = host_call(multi, utf8, off)
                    assert_same(got, ref, (opt, shape, prefix, pinned))
                if opt in ("tokens", "all_text"):
                    assert got["tok_offsets"] == e_off.tobytes() and got["tokens"] == e_toks.tobytes()


@pytest.mark.parametrize("n", SIZES)
def test_every_output_and_shape_device_resident(golden, golden_dict, n):
    """Device-resident batches: every last_device_* accessor (arrays or refusal) against the single device's, on
    every option set and batch shape, twice."""
    d, od, _ = golden_dict
    multi = vb.Tokenizer.new(d, devices=shard_devices(n))
    single = vb.Tokenizer.new(d)
    for opt in OPTIONS:
        configured(multi, opt)
        configured(single, opt)
        for shape, sents in shapes(golden).items():
            for prefix in (0, 3) if shape in ("mixed", "gaps") else (0,):
                utf8, off = pack(sents, prefix)
                ref = device_call(single, utf8, off)
                for _ in range(2):
                    assert_same(device_call(multi, utf8, off), ref, (opt, shape, prefix))
                if opt == "tokens":
                    e_off, e_toks, _ = od.tokenize_batch(*adv.pack(sents))
                    assert ref["tokens"] == (e_off.tobytes(), e_toks.tobytes())


def bounded_batch(golden, od, r):
    sents = golden_sents(golden) * 4 + [c["input"] for c in golden["tokenizer_cases"]]
    so = SpanOracle(od, r["char.def"], r["unk.def"], False, 0)
    spans, bounds = make_spans(so, sents, 3)
    spans[-1] = [(0, 6, "名詞,固有名詞")] if sents[-1].startswith("京都") else spans[-1]
    return sents, bounds, spans


@pytest.mark.parametrize("n", SIZES)
def test_bounded_and_span_calls(golden, golden_dict, n):
    """Boundaries and required tokens (with patterns), host and device-resident: a later shard's boundary and span
    lists start in the middle of the arrays.  Every output on."""
    d, od, r = golden_dict
    sents, bounds, spans = bounded_batch(golden, od, r)
    assert sum(map(len, spans)) > 10 and sum(map(len, bounds)) > 10 and any(len(x) > 2 for s in spans for x in s)
    utf8, off = adv.pack(sents)
    multi = configured(vb.Tokenizer.new(d, devices=shard_devices(n)), "all_text")
    single = configured(vb.Tokenizer.new(d), "all_text")
    for kw in (dict(boundaries=bounds), dict(spans=spans), dict(boundaries=bounds, spans=spans)):
        ref = host_call(single, utf8, off, **kw)
        for _ in range(2):
            assert_same(host_call(multi, utf8, off, **kw), ref, list(kw))
    configured(multi, "all")
    configured(single, "all")
    for kw in (dict(bounds=bounds), dict(spans=spans), dict(bounds=bounds, spans=spans)):
        ref = device_call(single, utf8, off, **kw)
        for _ in range(2):
            assert_same(device_call(multi, utf8, off, **kw), ref, list(kw))


# ---- input errors -------------------------------------------------------------------------------------------------------

def good_after(multi, single, utf8, off):
    """A good call on the tokenizer that just refused one still matches the single device."""
    assert_same(host_call(multi, utf8, off), host_call(single, utf8, off), "after an error")
    assert_same(device_call(multi, utf8, off), device_call(single, utf8, off), "after an error")


@pytest.mark.parametrize("n", SIZES)
def test_input_errors_match_single_device(golden, golden_dict, n):
    """Each input error gives the single device's status and message whichever shard holds it, also when several
    shards hold errors of different kinds (one device reports bad offsets, then invalid UTF-8, then bad boundaries,
    then bad spans)."""
    d, od, r = golden_dict
    sents = ["京都東京都京都", "東京都", "abc", "京都"] * 5
    assert len(sents) == 20
    utf8, off = adv.pack(sents)
    cut = cuts(off, n)
    assert cut[1] > 1 and cut[-2] < 19  # sentence 0 in the first shard, sentence 19 in the last
    multi = configured(vb.Tokenizer.new(d, devices=shard_devices(n)), "all")
    single = configured(vb.Tokenizer.new(d), "all")
    bad_utf8 = utf8.copy()
    bad_utf8[int(off[19])] = 0xFF  # never a UTF-8 byte
    ok_b, ok_s = [[] for _ in sents], [[] for _ in sents]
    bad_b_last = ok_b[:19] + [[100]]
    bad_b_first = [[100]] + ok_b[1:]
    bad_s_last = ok_s[:19] + [[(0, 100)]]
    bad_s_first = [[(0, 100)]] + ok_s[1:]
    down = off.copy()  # decreases inside the first shard (sentence 0 ends before it starts)
    down[1] = 0
    down[0] = 1
    cases = [
        ("utf8 last", bad_utf8, off, {}),
        ("bound last", utf8, off, dict(boundaries=bad_b_last)),
        ("span last", utf8, off, dict(spans=bad_s_last)),
        ("bound first, utf8 last", bad_utf8, off, dict(boundaries=bad_b_first)),
        ("span first, bound last", utf8, off, dict(spans=bad_s_first, boundaries=bad_b_last)),
        ("span first, utf8 last", bad_utf8, off, dict(spans=bad_s_first)),
        ("offsets first, utf8 last", bad_utf8, down, {}),
        ("bound first, offsets first", utf8, down, dict(boundaries=bad_b_first)),
    ]
    for c in cut[1:-1]:  # offsets that decrease at each cut: the sentence before it ends before it starts, and with 0
        if 0 < c < len(sents):  # there, before the shard does
            for end in (off[c - 1] - np.uint64(1), np.uint64(0)):
                o = off.copy()
                o[c] = end
                cases.append((f"decrease to {end} at cut {c}", utf8, o, {}))
                cases.append((f"decrease to {end} at cut {c}, utf8 last", bad_utf8, o, {}))
    for what, u, o, kw in cases:
        want = error_of(lambda: single.tokenize_batch(utf8=u, byte_offsets=o, **kw))
        assert error_of(lambda: multi.tokenize_batch(utf8=u, byte_offsets=o, **kw)) == want, ("host", what)
        dkw = {"bounds" if k == "boundaries" else k: v for k, v in kw.items()}
        want = error_of(lambda: device_call(single, u, o, **dkw))
        assert error_of(lambda: device_call(multi, u, o, **dkw)) == want, ("device", what)
        good_after(multi, single, utf8, off)


@pytest.mark.parametrize("n", SIZES)
def test_device_offsets_past_n_bytes_are_refused(golden_dict, n):
    """Device offsets that end beyond n_bytes are refused like on one device.  The input is a prefix of a larger
    device allocation, so that the bytes beyond n_bytes exist: a shard that sized its copy from the offsets alone
    would tokenize them."""
    d, _, _ = golden_dict
    sents = ["京都東京都京都", "東京都", "abc", "京都"] * 5
    utf8, off = adv.pack(sents)
    multi = configured(vb.Tokenizer.new(d, devices=shard_devices(n)), "all")
    single = configured(vb.Tokenizer.new(d), "all")
    for n_bytes in (len(utf8) - 1, int(off[10]), 0):
        want = error_of(lambda: device_call(single, utf8, off, n_bytes=n_bytes))
        assert "byte_offsets must be non-decreasing and end within the input buffer" in want[1]
        assert error_of(lambda: device_call(multi, utf8, off, n_bytes=n_bytes)) == want, n_bytes
        good_after(multi, single, utf8, off)


@pytest.mark.parametrize("n", SIZES)
def test_sample_base_limit(golden_dict, n):
    """sample_base + n_sent = 2^32 is the last accepted index range; one more is refused, like on one device."""
    d, _, _ = golden_dict
    sents = ["京都東京都京都", "東京都", "abc", ""] * 3
    utf8, off = adv.pack(sents)
    multi = configured(vb.Tokenizer.new(d, devices=shard_devices(n)), "samples")
    single = configured(vb.Tokenizer.new(d), "samples")
    for t in (multi, single):
        t.sample_base(2 ** 32 - len(sents))
    ref = host_call(single, utf8, off)
    assert_same(host_call(multi, utf8, off), ref, "host at 2^32")
    assert_same(device_call(multi, utf8, off), device_call(single, utf8, off), "device at 2^32")
    for t in (multi, single):
        t.sample_base(2 ** 32 - len(sents) + 1)
    want = error_of(lambda: single.tokenize_batch(utf8=utf8, byte_offsets=off))
    assert error_of(lambda: multi.tokenize_batch(utf8=utf8, byte_offsets=off)) == want
    want = error_of(lambda: device_call(single, utf8, off))
    assert error_of(lambda: device_call(multi, utf8, off)) == want
    for t in (multi, single):
        t.sample_base(0)
    good_after(multi, single, utf8, off)


# ---- counters, Worker, CLI ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", SIZES)
def test_counters(golden, golden_dict, n):
    """The "counting" counters and the connection-id counts add up over the shards to the single device's."""
    d, _, _ = golden_dict
    sents = shapes(golden)["mixed"]
    utf8, off = adv.pack(sents)
    multi = vb.Tokenizer.new(d, devices=shard_devices(n))
    single = vb.Tokenizer.new(d)
    for t in (multi, single):
        t.set_counting(True)
        t.tokenize_batch(utf8=utf8, byte_offsets=off)
    assert multi.last_counters().tolist() == single.last_counters().tolist()
    assert single.last_counters().any()
    multi, single = vb.Tokenizer.new(d, devices=shard_devices(n)), vb.Tokenizer.new(d)
    for t in (multi, single):
        t.init_connid_counter()
        t.tokenize_batch(utf8=utf8, byte_offsets=off)
        t.tokenize_batch(utf8=utf8, byte_offsets=off)
    for a, b in zip(multi.connid_counts(), single.connid_counts()):
        np.testing.assert_array_equal(a, b)


def test_worker_on_sharded_tokenizer(golden, golden_dict):
    d, _, _ = golden_dict
    multi = configured(vb.Tokenizer.new(d, devices=shard_devices(3)), "all")
    single = configured(vb.Tokenizer.new(d), "all")
    for s in golden_sents(golden):
        got = []
        for t in (multi, single):
            w = t.new_worker()
            w.reset_sentence(s)
            w.tokenize()
            got.append(([(x.surface(), x.feature(), x.total_cost(), x.prob()) for x in w.token_iter()],
                        [(x.surface(), x.margin(), x.prob()) for x in w.node_iter()], w.entropy(), w.log_path_prob(),
                        list(w.boundary_probs()), [w.posterior_token(i).surface() for i in range(w.num_posterior_tokens())],
                        [[x.surface() for x in w.sample_tokens(j)] for j in range(N_SAMP)]))
        assert got[0] == got[1], s


def test_tokenize_cli_repeated_devices(golden, tmp_path):
    """`tokenize --devices 0,0` and `0,0,0 --batch-lines 3` print what one device prints, in every mode."""
    exe = os.path.join(ROOT, "vibrato_b200", "bin", "tokenize")
    if not os.path.exists(exe):
        pytest.skip("CLIs not built")
    for k, v in golden["resources"].items():
        (tmp_path / k).write_text(v, encoding="utf-8", newline="")
    lines = ["京都東京都京都", "東京 都", "", "kampersanda", "東京県に行く", "", "京都 東京", "アイアイウ"] * 3
    text = ("\n".join(lines) + "\n").encode()
    base = [exe, "-i", str(tmp_path), "-u", str(tmp_path / "user.csv")]
    modes = [["-O", "mecab"], ["-O", "wakati"], ["-O", "detail"], ["-m", "-t", "0.01", "-O", "mecab"],
             ["-a", "-O", "mecab"], ["--sample", "3", "-t", "0.01", "--seed", "5", "-O", "wakati"],
             ["--posterior", "1", "-m", "-t", "0.01", "-O", "mecab"]]
    for mode in modes:
        ref = subprocess.run(base + mode, input=text, capture_output=True, timeout=120)
        assert ref.returncode == 0, ref.stderr.decode()
        assert ref.stdout.count(b"\n") >= len(lines)
        for flags in (["--devices", ",".join(map(str, shard_devices(2)))],
                      ["--devices", ",".join(map(str, shard_devices(3))), "--batch-lines", "3"]):
            p = subprocess.run(base + mode + flags, input=text, capture_output=True, timeout=120)
            assert p.returncode == 0, p.stderr.decode()
            assert p.stdout == ref.stdout, (mode, flags)
