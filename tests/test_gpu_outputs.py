"""Every batch output at once (tokens, marginals, lattice, samples and text) on every route, and the chunked
pipeline's host result growing past its initial estimates while keeping what it already holds."""
import string

import numpy as np
import pytest

import adversarial as adv
import vibrato_b200 as vb
from test_gpu_marginals import d2h, golden_dicts, golden_sents, skip_multi

pytestmark = pytest.mark.gpu
THETA = 0.001
N_SAMP = 3
ROUTES = ("whole", "chunked", "device", "multi", "multi_device")
NAMES = ("tok_offsets", "tokens", "token_probs", "path_probs", "node_offsets", "nodes", "node_links", "node_probs",
         "sample_offsets", "samples")


def make(d, route, text=True):
    tok = vb.Tokenizer.new(d, devices=[0, 1]) if route.startswith("multi") else vb.Tokenizer.new(d)
    if route == "chunked":
        tok.set_option("chunk_sentences", 64)
    tok.marginals(THETA).lattice(True).sampling(N_SAMP, THETA, 7)
    return tok.output_mode("mecab") if text else tok


def run(tok, route, sents, text=True):
    """{array name: array} of one call on `route`, with "text" on the host routes when `text`."""
    utf8, off = adv.pack(sents)
    n = len(sents)
    if route in ("device", "multi_device"):
        import torch
        d_utf8 = torch.from_numpy(utf8.copy() if len(utf8) else np.zeros(1, np.uint8)).cuda()
        d_off = torch.from_numpy(off.astype(np.int64)).cuda()
        torch.cuda.synchronize()
        a, b, nt = tok.tokenize_batch_device(d_utf8.data_ptr(), d_off.data_ptr(), n, len(utf8))
        tp, pp = tok.last_device_marginals()
        no, nodes, links, nprob, nn = tok.last_device_lattice()
        so, s, ns = tok.last_device_samples()
        arrays = (d2h(a, n + 1, np.uint64), d2h(b, nt, vb.TOKEN_DTYPE), d2h(tp, nt, np.float32), d2h(pp, n, np.float32),
                  d2h(no, n + 1, np.uint64), d2h(nodes, nn, vb.TOKEN_DTYPE), d2h(links, nn, vb.LINK_DTYPE),
                  d2h(nprob, nn, np.float32), d2h(so, n * N_SAMP + 1, np.uint64), d2h(s, ns, vb.TOKEN_DTYPE))
        return dict(zip(NAMES, arrays))
    res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
    got = {name: getattr(res, name).copy() for name in NAMES}
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


@pytest.mark.parametrize("route", ROUTES)
def test_all_outputs_on_every_route(golden, route):
    """Marginals, lattice, three samples and mecab text together: every array is byte-identical to the whole
    batch's (the device routes produce no text)."""
    skip_multi(route)
    d, _, _ = golden_dicts(golden, True)
    sents = golden_sents(golden) * 40 + [""] * 70 + golden_sents(golden) * 30  # empty runs across chunk edges
    ref = run(make(d, "whole"), "whole", sents)
    got = run(make(d, route), route, sents)
    assert ("text" in got) == (route not in ("device", "multi_device"))
    assert_same(got, ref)


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
