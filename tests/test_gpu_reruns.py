"""Every batch output at once (tokens, marginals, uncertainty with boundary probabilities, posterior paths, samples,
the lattice and the output text) through each way the engine aborts an attempt and runs the batch again: a candidate
pool, per-character slot count or chunk text buffer that outgrew its estimate, on every route that can hit it; the
chunked host result growing past its estimates in every record group but the text; and input errors in different
chunks, alone or beside an overflow, which every route reports like the whole batch.

Each case asserts, through describe()["last_reruns"], that the re-run it targets happened (and that the reference call
re-ran nothing), that every array is byte-identical to a whole-batch call sized large enough from the start, that the
tokenizer's next call on another batch equals a fresh tokenizer's, and that the sentences on either side of every
chunk cut match the restatements."""
import functools

import numpy as np
import pytest

import adversarial as adv
import format_oracle as fo
import lattice_oracle as lo
import margin_oracle as mg
import marginal_oracle as mo
import posterior_oracle as po
import sampling_oracle as so
import uncertainty_oracle as uo
import vibrato_b200 as vb
from bounded_oracle import BoundedOracle, vo_dictionary
from test_gpu_marginals import d2h, shard_devices
from test_gpu_sampling import check_parity
from test_gpu_shards import device_call as device_call_bounded, error_of
from test_gpu_uncertainty import close64
from oracle import vibrato_oracle as vo

pytestmark = pytest.mark.gpu
THETA = 0.01
N_SAMP = 3
SEED = 11
BIG_GAMMA = 200.0
MARGIN = 12
LETTERS = "abcdefghijklmnopqrstuvwxyz"
KANA = "あいうえおかきくけこさしすせそたちつてと"

# Two homographs per letter and a word for every letter pair: a run of letters is cheapest as pairs (the best path),
# while each single letter carries more probability than the pair over it (so the posterior path splits the pairs
# and has about twice the tokens).  About four candidates per byte; kana are grouped unknown words (DEFAULT).
LEX = "".join(f"{c},0,0,10,s0\n{c},0,0,12,s1\n" for c in LETTERS) + "".join(
    f"{a}{b},0,0,15,p\n" for a in LETTERS for b in LETTERS)
MATRIX = "1 1\n0 0 0\n"
CHAR_DEF = "DEFAULT 0 1 0\nSPACE 0 1 0\nALPHA 1 1 0\n\n0x0020 SPACE\n0x0061..0x007A ALPHA\n"
UNK_DEF = "DEFAULT,0,0,100,sym\nSPACE,0,0,100,space\nALPHA,0,0,1000,alpha\n"

# Chunked calls: chunk_sentences = 64 makes chunks of 1024 sentences and more, so a batch of 4096 runs as the three
# chunks [0, 1024) [1024, 2560) [2560, 4096) (engine.cu run_host).
N_SENT = 4096
CUTS = (0, 1024, 2560, 4096)
BIG_PERMILLE = 20000  # candidates per input byte (x 1000) no batch here reaches: no pool overflow
FMT_BIG = ("%m\\t%S\\n",)  # the whole sentence per token: far more text per byte than any learned ratio
FMT_PROB = ("%m\\t%pP\\t%S\\n",)


def checked(n):
    """The sentences restated in a batch of n: the first ones, both sides of every chunk cut, the last one."""
    return sorted({i for i in {0, 1, n - 1} | {c + k for c in CUTS[1:-1] for k in (-2, -1, 0, 1)} if 0 <= i < n})


@functools.lru_cache(maxsize=None)
def dicts():
    d = vb.SystemDictionaryBuilder.from_readers(LEX, MATRIX, CHAR_DEF, UNK_DEF)
    od = vo_dictionary(LEX, MATRIX, CHAR_DEF, UNK_DEF)
    return d, od, BoundedOracle(od, CHAR_DEF, UNK_DEF)


def word(rng, lo_, hi):
    return "".join(rng.choice(list(LETTERS), int(rng.integers(lo_, hi))))


def kana(rng, n):
    return "".join(rng.choice(list(KANA), n))


@functools.lru_cache(maxsize=None)
def pools(seed):
    """(dense, sparse): 150 distinct sentences of 9-13 letter words (about 250 candidates each), and 150 of a kana run
    and one short word (about 10), some of them empty."""
    rng = np.random.default_rng([seed, 31])
    dense = [" ".join(word(rng, 2, 7) for _ in range(int(rng.integers(9, 14)))) for _ in range(150)]
    sparse = [kana(rng, int(rng.integers(1, 6))) + " " + word(rng, 1, 3) for _ in range(140)] + [""] * 10
    return dense, sparse


def batch(dense_chunk, seed=0, n=N_SENT):
    """n sentences: chunk `dense_chunk` of CUTS holds the dense sentences, the rest the sparse ones.  A dense chunk has
    far more than the 2^16 candidates a pool sized at 1 per mille holds; the others far fewer."""
    dense, sparse = pools(seed)
    out = []
    for c in range(len(CUTS) - 1):
        src = dense if c == dense_chunk else sparse
        out += [src[(i * 7) % len(src)] for i in range(CUTS[c], min(CUTS[c + 1], n))]
    return tuple(out)


OTHER = batch(1, seed=5, n=1700)  # the second call of every case: other sentences, two chunks on a chunked route

# What a tokenizer renders and which lattice it keeps: (text source, lattice margin, posterior gamma)
SETUPS = {
    "best": ("best", None, 1.0),
    "lattice": ("lattice", None, BIG_GAMMA),
    "sample": ("sample", MARGIN, 1.0),
    "posterior": ("posterior", MARGIN, BIG_GAMMA),
}


def configure(tok, setup, style):
    src, margin, gamma = SETUPS[setup]
    tok.marginals(THETA).uncertainty(True, boundary_probs=True)
    tok.posterior(gamma, text=src == "posterior").sampling(N_SAMP, THETA, SEED, text=src == "sample")
    tok.lattice(True, text=src == "lattice", margin=margin)
    if style is None:
        return tok
    return tok.output_mode(style) if isinstance(style, str) else tok.output_format(*style)


def make(route, setup, style, **options):
    d, _, _ = dicts()
    tok = vb.Tokenizer.new(d, devices=shard_devices(2)) if route == "multi" else vb.Tokenizer.new(d)
    if route in ("chunked", "dual"):
        tok.set_option("chunk_sentences", 64)
    if route == "dual":
        tok.set_option("dual_stream", 1)
    for name, value in options.items():
        tok.set_option(name, value)
    return configure(tok, setup, style)


HOST = ("tok_offsets", "tokens", "token_probs", "path_probs", "entropies", "log_path_probs", "boundary_offsets",
        "boundary_probs", "node_offsets", "nodes", "node_links", "node_probs", "node_margins", "sample_offsets",
        "samples", "posterior_offsets", "posterior_tokens", "posterior_probs", "posterior_gains")


def device_call(tok, sents):
    """Every array of a tokenize_batch_device call, read through the last_device_* accessors."""
    import torch
    utf8, off = adv.pack(sents)
    n = len(sents)
    d_utf8 = torch.from_numpy(utf8.copy() if len(utf8) else np.zeros(1, np.uint8)).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    torch.cuda.synchronize()
    a, b, nt = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), n, len(utf8))
    tp, pp = tok.last_device_marginals()
    ent, lpp, boff, bprob, npos = tok.last_device_uncertainty()
    no, nodes, links, nprob, nn = tok.last_device_lattice()
    so_, s, ns = tok.last_device_samples()
    poff, ptok, pprob, pgain, npost = tok.last_device_posterior()
    got = dict(tok_offsets=d2h(a, n + 1, np.uint64), tokens=d2h(b, nt, vb.TOKEN_DTYPE), token_probs=d2h(tp, nt, np.float32),
               path_probs=d2h(pp, n, np.float32), entropies=d2h(ent, n, np.float64), log_path_probs=d2h(lpp, n, np.float64),
               boundary_offsets=d2h(boff, n + 1, np.uint64), boundary_probs=d2h(bprob, npos, np.float32),
               node_offsets=d2h(no, n + 1, np.uint64), nodes=d2h(nodes, nn, vb.TOKEN_DTYPE),
               node_links=d2h(links, nn, vb.LINK_DTYPE), node_probs=d2h(nprob, nn, np.float32),
               sample_offsets=d2h(so_, n * N_SAMP + 1, np.uint64), samples=d2h(s, ns, vb.TOKEN_DTYPE),
               posterior_offsets=d2h(poff, n + 1, np.uint64), posterior_tokens=d2h(ptok, npost, vb.TOKEN_DTYPE),
               posterior_probs=d2h(pprob, npost, np.float32), posterior_gains=d2h(pgain, n, np.float64))
    if tok._lattice_margin >= 0:
        got["node_margins"] = d2h(tok.last_device_lattice_margins(), nn, np.int64)
    return got


def call(tok, route, sents, **kw):
    """({array name: array}, "text" included on the host routes with an output stage; describe()["last_reruns"])."""
    if route == "device":
        return device_call(tok, sents), tok.describe()["last_reruns"]
    res = tok.tokenize_batch(sents, **kw)
    got = {name: getattr(res, name).copy() for name in HOST if getattr(res, name) is not None}
    if tok._format is not None or tok._options.get("output_mode"):
        got["text"] = res.text()
    res.close()
    return got, tok.describe()["last_reruns"]


NONE = {"pool": 0, "slots": 0, "text": 0}


@functools.lru_cache(maxsize=None)
def reference(setup, style, sents, spans=False):
    """A whole-batch call whose estimates are large enough from the start: nothing re-runs."""
    tok = make("whole", setup, style, pool_estimate_permille=BIG_PERMILLE)
    got, reruns = call(tok, "whole", list(sents), **span_args(sents, spans))
    assert reruns == NONE, reruns
    return got


def span_args(sents, spans):
    """Required tokens on the first letter of every dense sentence, with a boundary after its first word."""
    if not spans:
        return {}
    dense = [bool(s) and s[0] in LETTERS for s in sents]
    return dict(spans=[[(0, 1)] if x else [] for x in dense],
                boundaries=[[len(s.split(" ")[0])] if x else [] for s, x in zip(sents, dense)])


def assert_same(got, ref, what):
    want = {k for k in ref if k != "text"}
    assert {k for k in got if k != "text"} == want, what
    for name in want:
        assert got[name].tobytes() == ref[name].tobytes(), (what, name)
    if "text" in got:
        assert got["text"][1] == ref["text"][1], what
        np.testing.assert_array_equal(got["text"][0], ref["text"][0], err_msg=what)


def piece(off, recs, a, b):
    """Records a..b of a ragged group and their offsets rebased to 0."""
    return (off[a:b + 1] - off[a]).astype(np.uint64), recs[int(off[a]):int(off[b])]


def restate(got, sents, setup, style):
    """The CHECKED sentences of `got` against the restatements."""
    _, od, bo = dicts()
    src, margin, gamma = SETUPS[setup]
    for i in checked(len(sents)):
        s = sents[i].encode()
        what = (setup, i, sents[i])
        toff, toks = piece(got["tok_offsets"], got["tokens"], i, i + 1)
        assert toks.tobytes() == bo.tokenize(s).tobytes(), what
        noff, nodes = piece(got["node_offsets"], got["nodes"], i, i + 1)
        links = got["node_links"][int(got["node_offsets"][i]):int(got["node_offsets"][i + 1])]
        nprob = got["node_probs"][int(got["node_offsets"][i]):int(got["node_offsets"][i + 1])]
        boff, bprob = piece(got["boundary_offsets"], got["boundary_probs"], i, i + 1)
        poff, ptok = piece(got["posterior_offsets"], got["posterior_tokens"], i, i + 1)
        pprob = got["posterior_probs"][int(got["posterior_offsets"][i]):int(got["posterior_offsets"][i + 1])]
        soff, samples = piece(got["sample_offsets"], got["samples"], i * N_SAMP, (i + 1) * N_SAMP)
        check_parity(bo, [sents[i]], (soff, samples), N_SAMP, THETA, SEED,
                     expected=[so.sentence_samples(bo, s, N_SAMP, THETA, SEED, i)])
        ent, lpp, bnd = uo.sentence_uncertainty(bo, s, THETA)
        close64([got["entropies"][i], got["log_path_probs"][i]], [ent, lpp])
        mo.assert_f32_close(bprob, bnd, what=what)
        tp, pp = mo.sentence_marginals(bo, s, THETA)
        mo.assert_f32_close(got["token_probs"][int(got["tok_offsets"][i]):int(got["tok_offsets"][i + 1])], tp, what=what)
        mo.assert_f32_close(got["path_probs"][i:i + 1], [pp], what=what)
        if margin is None:
            e_nodes, e_links, e_probs = lo.sentence_lattice(bo, s, theta=THETA)
        else:
            e_nodes, e_links, e_margins, e_probs = mg.pruned_lattice(bo, s, margin, theta=THETA)
            m = got["node_margins"][int(got["node_offsets"][i]):int(got["node_offsets"][i + 1])]
            assert m.tobytes() == e_margins.tobytes(), what
        assert nodes.tobytes() == e_nodes.tobytes() and links.tobytes() == e_links.tobytes(), what
        mo.assert_f32_close(nprob, e_probs or [], what=what)
        if s and margin is None:  # bit for bit, fed the device's own marginals of every node
            lat = mo.Lattice(bo, s)
            order = [(e, k) for e in range(1, len(lat.ends)) for k in range(len(lat.ends[e]))]
            path, v = po.sweep(lat, dict(zip(order, nprob)), gamma)
            assert ptok.tobytes() == po.records(lat, path).tobytes(), what
            assert pprob.tobytes() == np.array([nprob[order.index(n)] for n in path], dtype=np.float32).tobytes()
            assert got["posterior_gains"][i] == v, what
        if "text" in got and style != FMT_PROB:  # the restatement prints no %pP
            utf8, off = vb.Tokenizer.pack([sents[i]] * (N_SAMP if src == "sample" else 1))
            recs = {"best": (toff, toks), "lattice": (noff, nodes), "posterior": (poff, ptok), "sample": (soff, samples)}[src]
            if isinstance(style, str):
                eoff, etext = vo.format_batch(od, utf8, off, *recs, style)
            else:
                eoff, etext = fo.format_batch(od, fo.Format(*style), utf8, off, *recs)
            toff_, text = got["text"]
            assert text[int(toff_[i]):int(toff_[i + 1])] == etext, what


def check_case(route, setup, style, reason, sents, spans=False, **options):
    """One call through `route` that must re-run for `reason` (or for nothing: None), against the reference, the
    restatements and, on the same tokenizer, a second call on OTHER."""
    sents = tuple(sents)
    tok = make(route, setup, style, **options)
    got, reruns = call(tok, route, list(sents), **span_args(sents, spans))
    want = dict(NONE)
    if reason:
        assert reruns[reason] >= 1, (reason, reruns)
        want[reason] = reruns[reason]
    assert reruns == want, reruns
    ref = reference(setup, style if route != "device" else None, sents, spans)
    assert_same(got, ref, (route, setup, reason))
    if not spans:
        restate(got, list(sents), setup, style if route != "device" else None)
    # the learned estimates carry over and nothing else does: the next batch is a fresh tokenizer's
    again, _ = call(tok, route, list(OTHER))
    assert_same(again, reference(setup, style if route != "device" else None, OTHER), (route, setup, reason, "again"))


POOL_CASES = [  # (route, dense chunk, setup, spans)
    ("whole", 0, "best", False),
    ("device", 1, "lattice", False),
    ("chunked", 0, "sample", False),
    ("chunked", 1, "posterior", False),
    ("chunked", 2, "best", False),
    ("dual", 1, "lattice", False),
    ("multi", 2, "posterior", False),
    ("whole", 0, "sample", True),
]


@pytest.mark.parametrize("route, dense, setup, spans", POOL_CASES,
                         ids=[f"{r}-chunk{c}-{s}" + ("-spans" if sp else "") for r, c, s, sp in POOL_CASES])
def test_pool_overflow(route, dense, setup, spans):
    """A pool sized at 1 candidate per 1000 bytes (2^16 here): the batch, or the chunk or shard holding the dense
    sentences, overflows it and runs again sized from what it counted."""
    _, _, bo = dicts()
    sents = batch(dense)
    if route == "multi":  # 600 dense sentences after the sparse ones: the byte split gives the second shard nearly all
        sents = sents[:CUTS[2] + 600]
    lattice_nodes = functools.lru_cache(maxsize=None)(lambda s: len(lo.sentence_lattice(bo, s.encode())[0]))
    n_bytes = sum(len(s.encode()) for s in sents)
    half = np.searchsorted(np.cumsum([len(s.encode()) for s in sents]), n_bytes / 2)
    pool = max(1 << 16, int(n_bytes * 0.001) + 4096)  # tests/segment_fixtures.py want_cand
    assert sum(lattice_nodes(s) for s in sents[CUTS[dense]:CUTS[dense + 1]]) > 1.5 * pool
    if route == "multi":
        assert sum(lattice_nodes(s) for s in sents[:half]) < pool / 2 and sum(lattice_nodes(s) for s in sents[half:]) > 1.2 * pool
    check_case(route, setup, "mecab", "pool", sents, spans, pool_estimate_permille=1)


@pytest.mark.parametrize("route, setup", [("whole", "posterior"), ("chunked", "best"), ("device", "sample")])
def test_slot_overflow(route, setup):
    """Launches sized for 1 character per 1000 bytes: the batch (every chunk) holds more and runs again with one
    slot per byte."""
    check_case(route, setup, "mecab", "slots", batch(1), chars_estimate_permille=1, pool_estimate_permille=BIG_PERMILLE)


@pytest.mark.parametrize("setup, style", [("best", FMT_PROB), ("lattice", FMT_BIG), ("sample", FMT_BIG)])
def test_text_overflow(setup, style):
    """A fresh tokenizer sizes each chunk's text from a few bytes per input byte; a format that prints the sentence
    with every token (node, sample) overflows it in the chunk of long sentences."""
    check_case("chunked", setup, style, "text", batch(0), pool_estimate_permille=BIG_PERMILLE)


def test_posterior_text_overflow_after_best_path_text():
    """Posterior text is sized from the ratio the best path's text taught: at a large gamma the posterior path splits
    most letter pairs, with about 1.5 times the text, so the chunk of long sentences overflows and runs again.  The
    ratio is learned on a smaller batch, so that the text buffers are sized from it anew."""
    sents = batch(1)
    tok = make("chunked", "posterior", "mecab", pool_estimate_permille=BIG_PERMILLE)
    tok.posterior(BIG_GAMMA, text=False)
    _, reruns = call(tok, "chunked", list(batch(1, n=1700)))
    assert reruns == NONE, reruns
    tok.posterior(BIG_GAMMA, text=True)
    got, reruns = call(tok, "chunked", list(sents))
    assert reruns["text"] >= 1 and reruns["pool"] == reruns["slots"] == 0, reruns
    assert_same(got, reference("posterior", "mecab", sents), "posterior text")
    restate(got, list(sents), "posterior", "mecab")
    again, _ = call(tok, "chunked", list(OTHER))
    assert_same(again, reference("posterior", "mecab", OTHER), "again")


def test_result_grows_in_every_record_group():
    """A tokenizer that learned its ratios on kana (1 character per 3 bytes, one token per run) is given a batch whose
    first chunk is kana and whose later chunks add a short word to every sentence: each chunk stays within its
    launch estimates, but the host result runs short in the token, lattice, sample, boundary-probability and
    posterior groups, grows, and keeps what the earlier chunks put there."""
    rng = np.random.default_rng(3)
    learn = [kana(rng, 7) for _ in range(2000)]
    first = [kana(rng, 7) for _ in range(CUTS[1])]
    later = [kana(rng, 7) + " " + word(rng, 3, 4) for _ in range(N_SENT - CUTS[1])]
    sents = first + later
    tok = make("chunked", "best", None, pool_estimate_permille=BIG_PERMILLE)
    a, reruns = call(tok, "chunked", learn)
    assert reruns == NONE, reruns
    a_bytes = sum(len(s.encode()) for s in learn)
    tpb = max(0.02, float(a["tok_offsets"][-1]) / a_bytes * 1.1)  # engine.cu run_host: the learned ratios
    cpb = min(1.0, float(a["boundary_offsets"][-1] - len(learn)) / a_bytes * 1.10)
    npb = max(0.1, float(a["node_offsets"][-1]) / a_bytes * 1.1)
    got, reruns = call(tok, "chunked", sents)
    assert reruns == NONE, reruns
    n_bytes, n = sum(len(s.encode()) for s in sents), len(sents)
    estimate = {"tok_offsets": int(n_bytes * tpb) + 1024, "node_offsets": int(n_bytes * npb) + 1024,  # Totals{...}
                "sample_offsets": int(n_bytes * tpb * N_SAMP) + 1024, "boundary_offsets": int(n_bytes * cpb) + n + 1024,
                "posterior_offsets": int(n_bytes * tpb) + 1024}
    for name, est in estimate.items():
        assert int(got[name][-1]) > est, (name, int(got[name][-1]), est)
    assert_same(got, reference("best", None, tuple(sents)), "grown")
    restate(got, sents, "best", None)


# Input errors in different chunks of CUTS (sentence 100 of the chunk holds each): every route reports the one the whole
# batch reports, the first in the engine's order (bad offsets, bad UTF-8, bad boundaries, bad spans) wherever it lies,
# also where a chunk overflowed its candidate pool or text buffer on the same attempt.
ERROR_CASES = {  # name: (setup, style, dense chunk, options, {error: chunk}, the error reported)
    "bound0-utf8_2": ("best", "mecab", 1, dict(pool_estimate_permille=BIG_PERMILLE), dict(bound=0, utf8=2), "utf8"),
    "span1-bound2": ("best", "mecab", 1, dict(pool_estimate_permille=BIG_PERMILLE), dict(span=1, bound=2), "bound"),
    "pool0-utf8_2": ("best", "mecab", 0, dict(pool_estimate_permille=1), dict(utf8=2), "utf8"),
    "text0-bound2": ("lattice", FMT_BIG, 0, dict(pool_estimate_permille=BIG_PERMILLE), dict(bound=2), "bound"),
}
MESSAGES = {"utf8": "stream did not contain valid UTF-8", "bound": "required boundaries must be non-decreasing"}


def refused(route, case):
    """((status, message), describe()["last_reruns"]) of the case's call on a fresh tokenizer, and the tokenizer."""
    setup, style, dense, options, errors, _ = ERROR_CASES[case]
    sents = list(batch(dense))
    at = {kind: CUTS[c] + 100 for kind, c in errors.items()}
    utf8, off = vb.Tokenizer.pack(sents)
    if "utf8" in at:
        assert sents[at["utf8"]]
        utf8 = utf8.copy()
        utf8[int(off[at["utf8"]])] = 0xFF  # never a UTF-8 byte
    far = 1 << 20  # beyond every sentence's end
    kw = {}
    if "bound" in at:
        kw["boundaries"] = [[far] if i == at["bound"] else [] for i in range(len(sents))]
    if "span" in at:
        kw["spans"] = [[(0, far)] if i == at["span"] else [] for i in range(len(sents))]
    tok = make(route, setup, style, **options)
    if route == "device":
        err = error_of(lambda: device_call_bounded(tok, utf8, off, bounds=kw.get("boundaries"), spans=kw.get("spans")))
    else:
        err = error_of(lambda: tok.tokenize_batch(utf8=utf8, byte_offsets=off, **kw))
    return err, tok.describe()["last_reruns"], tok


@functools.lru_cache(maxsize=None)
def whole_error(case):
    err, _, _ = refused("whole", case)
    return err


@pytest.mark.parametrize("case", list(ERROR_CASES))
@pytest.mark.parametrize("route", ["whole", "chunked", "dual", "device", "multi"])
def test_input_errors_across_chunks(route, case):
    """The case's call is refused with the whole batch's status and message, and books no re-run (a refused call
    reports none); the tokenizer's next call, on OTHER, equals a fresh whole-batch call."""
    setup, style, _, _, _, reported = ERROR_CASES[case]
    err, reruns, tok = refused(route, case)
    assert MESSAGES[reported] in whole_error(case)[1]
    assert err == whole_error(case), (route, case)
    assert reruns == NONE, (route, case, reruns)
    style = style if route != "device" else None
    again, _ = call(tok, route, list(OTHER))
    assert_same(again, reference(setup, style, OTHER), (route, case, "again"))
