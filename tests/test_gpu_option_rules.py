"""The rules between the options that choose what the output text renders: the best path, the lattice nodes
("lattice" = 2), the samples ("sample_text") or the posterior path ("posterior_text").  At most one of them replaces
the best path, each needs what it renders (sampling, posterior decoding), an output format's %pP needs marginals and
%pb needs lattice text, and a prerequisite cannot be switched off while the text renders it.  Every order of switching
between the four sources is walked from every combination of prerequisites: each refusal is checked against its full
message, and after each accepted change the arrays a result carries (the BatchResult attributes that are set and the
vbt_result_* accessors that answer)."""
import ctypes as C
import itertools

import pytest

import vibrato_b200 as vb
from test_gpu_marginals import golden_dicts
from vibrato_b200._native import check, lib

pytestmark = pytest.mark.gpu
THETA = 0.01
N_SAMP = 2
SENTS = ["東京都に住む", "", "京都東京都京都", "ＸＹＺ１２３"]

CONFLICT = "{} text and {} text both replace the output text: set {} before setting {}"
NAME = {"lattice": "lattice", "sample_text": "sample", "posterior_text": "posterior"}
OFF = {"lattice": '"lattice" below 2', "sample_text": '"sample_text" to 0', "posterior_text": '"posterior_text" to 0'}
ON = {"lattice": "lattice = 2", "sample_text": "sample_text = 1", "posterior_text": "posterior_text = 1"}
PAIR = [("lattice", "posterior_text"), ("lattice", "sample_text"), ("posterior_text", "sample_text")]  # message order

# output text: none, a fixed mode, a format that prints marginals (%pP), one that prints best-path flags (%pb)
FORMATS = {None: None, "wakati": None, "pP": ("%m\t%pP\n", None, "", "EOS\n"), "pb": ("%pb%m\n", None, "", "EOS\n")}
# sample text with a format that prints %pP or %pb: the refusal names the directive
SAMPLE_FORMAT = {
    "pP": 'node format, byte 3: %pP has no value in sample text (option "sample_text" = 1): a sampled token has no marginal',
    "pb": 'node format, byte 0: %pb has no value in sample text (option "sample_text" = 1): a sampled token has no '
          "best-path flag"}
# a result's arrays: BatchResult attribute -> the accessor that answers for it
ACCESSORS = {"token_probs": "marginals", "nodes": "lattice", "node_probs": None, "samples": "samples",
             "entropies": "uncertainty", "boundary_probs": None, "posterior_tokens": "posterior"}


class State:
    """The options as the engine is expected to hold them, and what it is expected to say to each change."""

    def __init__(self, marg, samp, post, unc, fmt):
        self.marg, self.samp, self.post, self.unc, self.fmt = marg, samp, post, unc, fmt
        self.lattice, self.text = 0, None  # text: the option whose source renders the text, None = the best path

    def refusal(self, option, value):
        """The message the engine refuses option = value with, or None when it accepts it."""
        if option == "lattice":
            if value != 2 and self.fmt == "pb":
                return "the output format prints %pb, which only lattice text has: change the format before setting lattice below 2"
            if value == 2 and self.text not in (None, "lattice"):
                return self.conflict("lattice")
            return None
        if option == "sampling_off":
            return ('the output text renders the samples: set "sample_text" to 0 before switching sampling off'
                    if self.text == "sample_text" else None)
        if option == "posterior_off":
            return ('the output text renders the posterior path: set "posterior_text" to 0 before switching posterior '
                    "decoding off" if self.text == "posterior_text" else None)
        if option == "marginals_off":
            if self.fmt == "pP":
                return "the output format prints %pP: change the format before switching marginals off"
            if self.unc:
                return 'uncertainty needs marginals: set the option "uncertainty" to 0 before switching marginals off'
            if self.post:
                return "posterior decoding needs marginals: switch it off with set_posterior before switching marginals off"
            return None
        if not value:  # "sample_text" / "posterior_text" = 0
            return None
        if option == "sample_text" and self.fmt in SAMPLE_FORMAT:  # the C ABI compiles the format again first
            return SAMPLE_FORMAT[self.fmt]
        if option == "sample_text" and not self.samp:
            return "sample_text needs sampling: switch it on with set_sampling first"
        if option == "posterior_text" and not self.post:
            return "posterior_text needs posterior decoding: switch it on with set_posterior first"
        if self.text not in (None, option):
            return self.conflict(option)
        return None

    def conflict(self, option):
        first, second = next(p for p in PAIR if set(p) == {option, self.text})
        return CONFLICT.format(NAME[first], NAME[second], OFF[self.text], ON[option])

    def apply(self, option, value):
        if option == "lattice":
            self.lattice = value
            if value == 2:
                self.text = "lattice"
            elif self.text == "lattice":
                self.text = None
        elif option in ("sample_text", "posterior_text"):
            if value:
                self.text = option
            elif self.text == option:
                self.text = None

    def arrays(self):
        """The BatchResult attributes a result carries."""
        has = {"token_probs": self.marg, "nodes": self.lattice > 0, "node_probs": self.lattice > 0 and self.marg,
               "samples": self.samp, "entropies": self.marg and self.unc > 0, "boundary_probs": self.marg and self.unc > 1,
               "posterior_tokens": self.marg and self.post}
        return {k for k, v in has.items() if v}

    def accessors(self):
        """The vbt_result_* accessors that answer."""
        out = {ACCESSORS[a] for a in self.arrays() if ACCESSORS[a]}
        return out | ({"text"} if self.fmt else set())


def change(tok, state, option, value):
    """Asks the engine for option = value; checks its answer against the expected one and returns whether it took it."""
    expected = state.refusal(option, value)
    if expected is not None:
        refused(lambda: tok.set_option(option, value), expected)
        return False
    tok.set_option(option, value)
    state.apply(option, value)
    check_result(tok, state)
    return True


def refused(call, expected):
    with pytest.raises(vb.VibratoError) as e:
        call()
    assert e.value.code == 1 and str(e.value) == "InvalidArgument: " + expected


def check_result(tok, state):
    res = tok.tokenize_batch(SENTS)
    assert {a for a in ACCESSORS if getattr(res, a) is not None} == state.arrays()
    p = [C.c_void_p() for _ in range(5)]
    n = C.c_uint64()
    calls = {"marginals": lambda h: lib().vbt_result_marginals(h, C.byref(p[0]), C.byref(p[1])),
             "lattice": lambda h: lib().vbt_result_lattice(h, *[C.byref(x) for x in p[:4]], C.byref(n)),
             "samples": lambda h: lib().vbt_result_samples(h, C.byref(p[0]), C.byref(p[1]), C.byref(n)),
             "uncertainty": lambda h: lib().vbt_result_uncertainty(h, *[C.byref(x) for x in p[:4]]),
             "posterior": lambda h: lib().vbt_result_posterior(h, *[C.byref(x) for x in p[:4]], C.byref(n)),
             "text": lambda h: lib().vbt_result_text(h, C.byref(p[0]), C.byref(p[1]), C.byref(n))}
    assert {name for name, f in calls.items() if f(res._h) == 0} == state.accessors()
    res.close()


def prerequisites():
    for marg, samp, fmt in itertools.product((False, True), (False, True), FORMATS):
        for post, unc in itertools.product((False, True), (0, 2)) if marg else [(False, 0)]:
            if fmt != "pP" or marg:
                yield marg, samp, post, unc, fmt


def setup(tok, marg, samp, post, unc, fmt):
    """A tokenizer with every text option off, then the prerequisites (and for %pb the lattice text it needs)."""
    for name in ("sample_text", "posterior_text"):
        tok.set_option(name, 0)
    tok.output_format(None).output_mode(None).lattice(False).uncertainty(False).posterior(None).sampling(0).marginals(None)
    state = State(marg, samp, post, unc, fmt)
    tok.marginals(THETA if marg else None).sampling(N_SAMP if samp else 0, THETA, 7)
    tok.posterior(1.0 if post else None).uncertainty(unc > 0, boundary_probs=unc > 1)
    if fmt == "pb":
        tok.set_option("lattice", 2)
        state.apply("lattice", 2)
    if fmt == "wakati":
        tok.output_mode("wakati")
    elif fmt:
        tok.output_format(*FORMATS[fmt])
    return state


@pytest.fixture(scope="module")
def tok(golden):
    d, _, _ = golden_dicts(golden, True)
    return vb.Tokenizer.new(d)


SOURCES = {"best": None, "lattice": ("lattice", 2), "sample_text": ("sample_text", 1), "posterior_text": ("posterior_text", 1)}


def switch_off(tok, state):
    """Back to the best path from the current source (refused while %pb needs lattice text)."""
    if state.text == "lattice":
        return change(tok, state, "lattice", 1)
    if state.text:
        return change(tok, state, state.text, 0)
    return True


@pytest.mark.parametrize("prereq", list(prerequisites()), ids=lambda p: "marg{}-samp{}-post{}-unc{}-{}".format(*p))
def test_every_order_of_text_sources(tok, prereq):
    for order in itertools.permutations(SOURCES):
        state = setup(tok, *prereq)
        check_result(tok, state)
        for src in order:
            if SOURCES[src] is None:
                switch_off(tok, state)
                continue
            option, value = SOURCES[src]
            if not change(tok, state, option, value) and state.text not in (None, option):
                # refused for another source: switch that one off, then ask again
                if switch_off(tok, state):
                    change(tok, state, option, value)
            # a prerequisite cannot leave while the text renders it (or an output that needs it is on)
            h = tok.handle()
            for off, call in (("sampling_off", lambda: check(lib().vbt_tokenizer_set_sampling(h, 0, 0.0, 0))),
                              ("posterior_off", lambda: check(lib().vbt_tokenizer_set_posterior(h, 0, 0.0))),
                              ("marginals_off", lambda: check(lib().vbt_tokenizer_set_marginals(h, 0.0)))):
                if state.refusal(off, None) is not None:
                    refused(call, state.refusal(off, None))
