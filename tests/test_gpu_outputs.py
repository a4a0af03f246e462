"""Every batch output at once (tokens, marginals, uncertainty, lattice, node margins, samples, posterior paths and
text) on every route, the chunked pipeline's host result growing past its initial estimates while keeping what it
already holds, and the refusals of the device-resident accessors."""
import re
import string

import numpy as np
import pytest

import adversarial as adv
import vibrato_b200 as vb
from test_gpu_marginals import d2h, golden_dicts, golden_sents, shard_devices

pytestmark = pytest.mark.gpu
THETA = 0.001
N_SAMP = 3
ROUTES = ("whole", "chunked", "device", "multi", "multi_device")
NAMES = ("tok_offsets", "tokens", "token_probs", "path_probs", "entropies", "log_path_probs", "boundary_offsets",
         "boundary_probs", "node_offsets", "nodes", "node_links", "node_probs", "node_margins", "sample_offsets", "samples",
         "posterior_offsets", "posterior_tokens", "posterior_probs", "posterior_gains")
MARGIN = 2000  # the near-best lattice's cost margin when it is on


def make(d, route, text=True, margin=None):
    tok = vb.Tokenizer.new(d, devices=shard_devices(2)) if route.startswith("multi") else vb.Tokenizer.new(d)
    if route == "chunked":
        tok.set_option("chunk_sentences", 64)
    tok.marginals(THETA).uncertainty(True, boundary_probs=True).posterior(2.0)
    tok.lattice(True, margin=margin).sampling(N_SAMP, THETA, 7)
    return tok.output_mode("mecab") if text else tok


def device_call(tok, utf8, off):
    """tokenize_batch_device on the packed batch, its input on the first device."""
    import torch
    d_utf8 = torch.from_numpy(utf8.copy() if len(utf8) else np.zeros(1, np.uint8)).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    torch.cuda.synchronize()
    return tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), len(off) - 1, len(utf8))


def run(tok, route, sents, text=True, margin=None):
    """{array name: array} of one call on `route`, with "text" on the host routes when `text`, and "node_margins"
    when `margin` is set."""
    names = [name for name in NAMES if name != "node_margins" or margin is not None]
    utf8, off = adv.pack(sents)
    n = len(sents)
    if route in ("device", "multi_device"):
        a, b, nt = device_call(tok, utf8, off)
        tp, pp = tok.last_device_marginals()
        no, nodes, links, nprob, nn = tok.last_device_lattice()
        nm = tok.last_device_lattice_margins() if margin is not None else None
        so, s, ns = tok.last_device_samples()
        ent, lpp, boff, bprob, npos = tok.last_device_uncertainty()
        poff, ptok, pprob, pgain, npost = tok.last_device_posterior()
        arrays = (d2h(a, n + 1, np.uint64), d2h(b, nt, vb.TOKEN_DTYPE), d2h(tp, nt, np.float32), d2h(pp, n, np.float32),
                  d2h(ent, n, np.float64), d2h(lpp, n, np.float64), d2h(boff, n + 1, np.uint64),
                  d2h(bprob, npos, np.float32), d2h(no, n + 1, np.uint64), d2h(nodes, nn, vb.TOKEN_DTYPE),
                  d2h(links, nn, vb.LINK_DTYPE), d2h(nprob, nn, np.float32), None if nm is None else d2h(nm, nn, np.int64),
                  d2h(so, n * N_SAMP + 1, np.uint64), d2h(s, ns, vb.TOKEN_DTYPE), d2h(poff, n + 1, np.uint64),
                  d2h(ptok, npost, vb.TOKEN_DTYPE), d2h(pprob, npost, np.float32), d2h(pgain, n, np.float64))
        return {name: x for name, x in zip(NAMES, arrays) if name in names}
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
    got = {name: getattr(res, name).copy() for name in names}
    if text:
        got["text"] = res.text()
    res.close()
    return got


def assert_same(got, ref):
    for name, a in got.items():
        if name == "text":
            assert a[1] == ref[name][1]
            np.testing.assert_array_equal(a[0], ref[name][0])
        else:
            assert a.tobytes() == ref[name].tobytes(), name


def check_all_outputs(golden, route, margin):
    d, _, _ = golden_dicts(golden, True)
    sents = golden_sents(golden) * 40 + [""] * 70 + golden_sents(golden) * 30  # empty runs across chunk edges
    ref = run(make(d, "whole", margin=margin), "whole", sents, margin=margin)
    got = run(make(d, route, margin=margin), route, sents, margin=margin)
    assert ("text" in got) == (route not in ("device", "multi_device"))
    assert ("node_margins" in got) == (margin is not None)
    assert_same(got, ref)


@pytest.mark.parametrize("route", ROUTES)
def test_all_outputs_on_every_route(golden, route):
    """Marginals, uncertainty, lattice, three samples, posterior paths and mecab text together: every array is
    byte-identical to the whole batch's (the device routes produce no text)."""
    check_all_outputs(golden, route, None)


@pytest.mark.parametrize("route", ROUTES)
def test_all_outputs_with_lattice_margins_on_every_route(golden, route):
    """The same with the near-best lattice: its nodes and their margins are byte-identical on every route too."""
    check_all_outputs(golden, route, MARGIN)


def dense_dictionary():
    """Four homographs per lowercase letter and grouped unknown words for the rest: "a b c ..." is one token per byte
    and about three lattice nodes per byte."""
    lex = "".join(f"{c},0,0,{k + 1},w{k}\n" for c in string.ascii_lowercase for k in range(4))
    char = "DEFAULT 0 1 0\nSPACE 0 1 0\nALPHA 1 1 0\n\n0x0020 SPACE\n0x0061..0x007A ALPHA\n"
    unk = "DEFAULT,0,0,100,sym\nSPACE,0,0,100,space\nALPHA,0,0,100,alpha\n"
    return vb.SystemDictionaryBuilder.from_readers(lex, "1 1\n0 0 0\n", char, unk)


def test_chunked_result_grows_and_keeps():
    """A fresh tokenizer sizes its chunked host result for 0.2 tokens and 2 nodes per input byte.  The first chunk
    (1024 short sentences) fits; the later ones (long sentences of one token and about three nodes per byte) overflow
    the token, token_prob, node, link, node_prob and sample arrays, which grow and keep the first chunk's records."""
    d = dense_dictionary()
    letters = string.ascii_lowercase
    long_sent = " ".join(letters[i % 26] for i in range(100))
    sents = ["a b"] * 1024 + [long_sent] * 2000
    n_bytes = sum(len(s) for s in sents)
    ref = run(make(d, "whole", text=False), "whole", sents, text=False)
    got = run(make(d, "chunked", text=False), "chunked", sents, text=False)
    assert len(ref["tokens"]) > 0.2 * n_bytes + 1024
    assert len(ref["nodes"]) > 2 * n_bytes + 1024
    assert len(ref["samples"]) > 0.2 * n_bytes * N_SAMP + 1024
    assert_same(got, ref)


REFUSALS = {"last_device_marginals": "marginals", "last_device_lattice": "the lattice",
            "last_device_lattice_margins": "the lattice's cost margin", "last_device_samples": "sampling"}


@pytest.mark.parametrize("route", ("device", "multi_device"))
def test_last_device_accessors_refuse(golden, route):
    """Each last_device_* accessor names what the last device-resident call ran without: after a call made with none
    of the features, and after a call with every feature on that failed (invalid UTF-8)."""
    d, _, _ = golden_dicts(golden, True)
    utf8, off = adv.pack(["京都東京都京都", "abc"])

    def assert_refused(tok):
        for name, what in REFUSALS.items():
            with pytest.raises(vb.VibratoError, match=re.escape(f"the last device-resident call ran without {what}") + "$"):
                getattr(tok, name)()

    plain = vb.Tokenizer.new(d, devices=shard_devices(2)) if route == "multi_device" else vb.Tokenizer.new(d)
    device_call(plain, utf8, off)
    assert_refused(plain)
    full = make(d, route, text=False, margin=MARGIN)
    device_call(full, utf8, off)
    for name in REFUSALS:  # the same call with every feature on is served
        getattr(full, name)()
    bad = utf8.copy()
    bad[-2] = 0xFF  # never a UTF-8 byte
    with pytest.raises(vb.VibratoError, match="UTF-8"):
        device_call(full, bad, off)
    assert_refused(full)
