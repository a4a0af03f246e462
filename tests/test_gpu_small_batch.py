"""The one-launch route for small host batches (tokenizer option "small_batch", kernel k_small_batch).

Every call below goes through two tokenizers over the same dictionary, one with the option on and one without, and
compares both with the oracle: token records, offsets and, where the output stage is on, the text, byte for byte.
Calls that should take the new route also assert describe()["last_viterbi"] == "k_small_batch" and exactly one
kernel launch."""
import os
import pty
import subprocess
import termios

import numpy as np
import pytest

import adversarial as adv
import vibrato_b200 as vb
from oracle import vibrato_oracle as vo
from test_gpu_marginals import shard_devices

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("mecab", "wakati", "detail")
EAGER_BYTES = 16384  # the route's input limit (engine.cu kEagerBytes)


def assert_batch_equal(res, tok_off, toks):
    assert res.n_sent == len(tok_off) - 1
    np.testing.assert_array_equal(res.tok_offsets, tok_off)
    assert res.n_tokens == len(toks)
    for name in vb.TOKEN_DTYPE.names:
        np.testing.assert_array_equal(res.tokens[name], toks[name], err_msg=name)


class Pair:
    """A tokenizer with small_batch(n) and one on the default route, same dictionary and settings."""

    def __init__(self, d, od, ignore_space=False, max_grouping_len=0, n=64):
        self.od, self.ignore_space, self.mgl = od, ignore_space, max_grouping_len
        self.small = vb.Tokenizer.new(d).ignore_space(ignore_space).max_grouping_len(max_grouping_len).small_batch(n)
        self.ref = vb.Tokenizer.new(d).ignore_space(ignore_space).max_grouping_len(max_grouping_len)

    def set(self, fn):
        fn(self.small)
        fn(self.ref)

    def check(self, utf8, off, mode=None, route="k_small_batch"):
        """Both tokenizers on one batch, against the oracle; `route` = what the small tokenizer must report."""
        tok_off, toks = self.od.tokenize_batch(utf8, off, self.ignore_space, self.mgl)[:2]
        a = self.small.tokenize_batch(utf8=utf8, byte_offsets=off)
        assert self.small.describe()["last_viterbi"] == route
        if route == "k_small_batch":
            assert self.small.last_launch_count() == 1
            ms = self.small.last_stage_ms()
            assert ms["viterbi"] >= 0 and sum(v for k, v in ms.items() if k != "viterbi") == 0
        b = self.ref.tokenize_batch(utf8=utf8, byte_offsets=off)
        assert self.ref.describe()["last_viterbi"] != "k_small_batch"
        assert_batch_equal(a, tok_off, toks)
        assert_batch_equal(b, tok_off, toks)
        if a.compact is not None:
            assert a.compact.tobytes() == b.compact.tobytes()
        if mode is not None:
            eoff, etext = vo.format_batch(self.od, utf8, off, tok_off, toks, mode)
            for r in (a, b):
                toff, text = r.text()
                np.testing.assert_array_equal(toff, eoff)
                assert text == etext
        return a


def batches(sents, max_n, max_bytes=EAGER_BYTES):
    """Consecutive batches of at most max_n sentences and max_bytes bytes."""
    out, cur, size = [], [], 0
    for s in sents:
        n = len(s.encode())
        if cur and (len(cur) == max_n or size + n > max_bytes):
            out.append(cur)
            cur, size = [], 0
        cur.append(s)
        size += n
    if cur:
        out.append(cur)
    return out


def golden_pair(golden, user, **kw):
    r = golden["resources"]
    d = vb.SystemDictionaryBuilder.from_readers(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
    od = vo.OracleDictionary(r["lex.csv"], r["matrix.def"], r["char.def"], r["unk.def"])
    if user:
        d.reset_user_lexicon_from_reader(r["user.csv"])
        od.set_user_csv(r["user.csv"])
    return Pair(d, od, **kw)


def adversarial_pair(d, connector="matrix", **kw):
    if connector == "matrix":
        dev = vb.SystemDictionaryBuilder.from_readers(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    else:
        right, left, cost = d.matrix
        dev = vb.SystemDictionaryBuilder.from_readers_with_bigram_info(d.lex_csv, right, left, cost, d.char_def, d.unk_def,
                                                                       dual_connector=connector == "dual")
    od = vo.OracleDictionary(d.lex_csv, d.matrix, d.char_def, d.unk_def, dual_connector=connector == "dual")
    dev.reset_user_lexicon_from_reader(d.user_csv)
    od.set_user_csv(d.user_csv)
    return Pair(dev, od, **kw)


def test_golden_fixture_sentences(golden):
    cases = golden["tokenizer_cases"]
    settings = sorted({(c["user"], c["ignore_space"], c["max_grouping_len"]) for c in cases})
    for user, ignore_space, mgl in settings:
        p = golden_pair(golden, user, ignore_space=ignore_space, max_grouping_len=mgl)
        sents = [c["input"] for c in cases if (c["user"], c["ignore_space"], c["max_grouping_len"]) == (user, ignore_space, mgl)]
        for s in sents:  # one sentence per call
            p.check(*adv.pack([s]))
        p.check(*adv.pack(sents))  # and as one batch
        all_sents = [c["input"] for c in cases]
        for mode in MODES:
            p.set(lambda t: t.output_mode(mode))
            p.check(*adv.pack(all_sents), mode=mode)
            p.check(*adv.pack(all_sents[:1]), mode=mode)
        p.set(lambda t: t.output_mode(None))


@pytest.mark.parametrize("ignore_space", [False, True])
@pytest.mark.parametrize("dictionary", list(adv.FAMILIES) + ["raw", "dual"])
def test_adversarial_sentences(dictionary, ignore_space):
    """Every cost family on the Matrix connector and the wrapping bigram costs on Raw and Dual, with batches of 1 to
    64 sentences, sentences that end in spaces and sentences made only of spaces."""
    if dictionary in adv.FAMILIES:
        d, connector = adv.make_dictionary(dictionary), "matrix"
    else:
        d, connector = adv.make_dictionary("wrap", dual=dictionary == "dual"), dictionary
    p = adversarial_pair(d, connector, ignore_space=ignore_space)
    sents = adv.make_sentences(d, 400, seed=5, max_len=80)
    sents[10:10] = [" ", "   ", "a  ", "あ ア  ", "", " a"]
    assert any(s.endswith(" ") and s.strip() for s in sents)
    for n in (1, 7, 64):
        for batch in batches(sents, n)[:12]:
            p.check(*adv.pack(batch))
    p.set(lambda t: t.output_mode("detail"))
    p.check(*adv.pack(sents[:64]), mode="detail")


@pytest.mark.parametrize("mgl", [0, 1, 24])
def test_max_grouping_len_user_lexicon_compact_and_modes(mgl):
    d = adv.make_dictionary("ties", seed=3)
    p = adversarial_pair(d, ignore_space=True, max_grouping_len=mgl, n=100)
    sents = adv.make_sentences(d, 64, seed=11, max_len=120)
    sents += ["a" * 40 + "ア" * 30, "1" * 50, "漢" * 30 + " " * 3]  # long groupable runs
    utf8, off = adv.pack(sents)
    p.check(utf8, off)
    for mode in MODES:
        p.set(lambda t: t.output_mode(mode))
        p.check(utf8, off, mode=mode)
    p.set(lambda t: t.output_mode(None))
    p.set(lambda t: t.compact_tokens(True))
    p.check(utf8, off)
    p.check(*adv.pack(sents[:1]))


@pytest.mark.parametrize("w,c", [(32767, 32767), (-32768, -32768)])
def test_single_path_costs_near_the_i32_limit(w, c):
    """The single-path construction of test_gpu_viterbi_routes: 16 384 characters (all the route admits) reach
    +-1.07e9, checked against the closed form wrap_i32(k * (w + c)); `aa` next to `a` makes the search compare them."""
    n = EAGER_BYTES
    sents = ["a" * (n - 40), "a" * 7, "", " " + "a" * 20 + "  "]
    utf8, off = adv.pack(sents)
    assert len(utf8) <= EAGER_BYTES
    k = np.arange(1, n - 40 + 1, dtype=np.int64)
    closed = np.array([adv.wrap_i32(x) for x in k * (w + c)], dtype=np.int32)
    for ignore_space in (False, True):
        od = vo.OracleDictionary(*adv.single_word_dictionary(w, c))
        p = Pair(vb.SystemDictionaryBuilder.from_readers(*adv.single_word_dictionary(w, c)), od, ignore_space=ignore_space)
        res = p.check(utf8, off)
        np.testing.assert_array_equal(res.tokens["total_cost"][: n - 40], closed)
    for aa in (-32768, 0, 32767):
        src = adv.single_word_dictionary(w, c, with_aa=aa)
        p = Pair(vb.SystemDictionaryBuilder.from_readers(*src), vo.OracleDictionary(*src))
        p.check(utf8, off)


def test_threshold_dictionary():
    d = adv.threshold_dictionary()
    p = adversarial_pair(d, n=100)
    sents = adv.make_sentences(d, 30, seed=9, max_len=8)
    sents.insert(5, "z" * 16000)
    utf8, off = adv.pack(sents)
    assert len(utf8) <= EAGER_BYTES
    res = p.check(utf8, off)
    assert int(res.tokens["total_cost"][int(res.tok_offsets[6]) - 1]) == -65536 * 16000


def test_empty_sentences_and_empty_batch(golden):
    p = golden_pair(golden, True)
    for sents in ([], [""], ["", "", ""], ["", "東京都", "", "", "京都", ""]):
        p.check(*adv.pack(sents))
        for mode in MODES:
            p.set(lambda t: t.output_mode(mode))
            p.check(*adv.pack(sents), mode=mode)
        p.set(lambda t: t.output_mode(None))


def test_input_errors_then_a_good_call(golden):
    p = golden_pair(golden, False)
    good = adv.pack(["東京都", "京都"])
    bad_utf8 = (np.frombuffer("東京".encode() + b"\xff\xfe" + "都".encode(), dtype=np.uint8), np.array([0, 3, 11], dtype=np.uint64))
    decreasing = (np.frombuffer("東京都京都".encode(), dtype=np.uint8), np.array([0, 9, 3, 15], dtype=np.uint64))
    for mode in (None, "mecab"):
        p.set(lambda t: t.output_mode(mode))
        for utf8, off in (bad_utf8, decreasing):
            codes = []
            for t in (p.small, p.ref):
                with pytest.raises(vb.VibratoError) as e:
                    t.tokenize_batch(utf8=utf8, byte_offsets=off)
                codes.append(e.value.code)
            assert codes[0] == codes[1]
            p.check(*good, mode=mode)


def test_scratch_overflow_falls_back_to_the_usual_route():
    """More candidates than the route's pool (a word with 200 homographs, 1 000 times), and more text than its text
    buffer (2 000 one-character words with 1-2 KB features): the same result, from the usual route."""
    lex = "".join(f"a,0,0,{i % 7},A{i}\n" for i in range(200))
    src = (lex, "1 1\n0 0 0\n", "DEFAULT 0 1 0\n", "DEFAULT,0,0,30000,*\n")
    p = Pair(vb.SystemDictionaryBuilder.from_readers(*src), vo.OracleDictionary(*src))
    p.check(*adv.pack(["a" * 1000]), route="k_viterbi2")
    p.check(*adv.pack(["a" * 20]))  # the next small call takes the route again
    rng = np.random.default_rng(8)
    chars = "abcdefghijklmnop"
    lex = "".join(f"{c},0,0,{10 * i},{c}:" + "x" * int(rng.integers(1000, 2000)) + "\n" for i, c in enumerate(chars))
    src = (lex, "1 1\n0 0 0\n", "DEFAULT 0 1 0\n", "DEFAULT,0,0,30000,*\n")
    p = Pair(vb.SystemDictionaryBuilder.from_readers(*src), vo.OracleDictionary(*src))
    long_text = ["".join(rng.choice(list(chars), size=2000))]
    for mode in ("mecab", "detail"):
        p.set(lambda t: t.output_mode(mode))
        p.check(*adv.pack(long_text), mode=mode, route="k_viterbi2")
        p.check(*adv.pack(["abc", chars * 20]), mode=mode)  # more text than the first copy guessed: a second copy


def test_routing_limits(golden):
    p = golden_pair(golden, True, n=8)
    sents = ["東京都に行く", "京都", "", "kampersanda"] * 2
    p.check(*adv.pack(sents))  # 8 sentences: the route
    p.check(*adv.pack(sents + ["都"]), route="k_viterbi2")  # 9 > N
    big = ["東京都" * 1000, "京都" * 1300]  # 9 000 + 7 800 bytes
    assert len("".join(big).encode()) > EAGER_BYTES
    p.check(*adv.pack(big), route="k_viterbi2")
    p.check(*adv.pack(big[:1]))
    p.small.set_counting(True)  # counted runs stay on k_viterbi
    p.check(*adv.pack(sents), route="k_viterbi")
    p.small.set_counting(False)
    p.small.small_batch(0)  # off: exactly the default route
    utf8, off = adv.pack(sents)
    p.check(utf8, off, route="k_viterbi2")
    assert p.small.last_launch_count() == p.ref.last_launch_count() > 1
    with pytest.raises(vb.VibratoError):
        p.small.small_batch(-1)
    with pytest.raises(vb.VibratoError):
        p.small.small_batch(65537)


def test_worker_loop():
    d = adv.make_dictionary("extreme", seed=4)
    p = adversarial_pair(d, ignore_space=True)
    sents = adv.make_sentences(d, 500, seed=21, max_len=60)
    got = []
    for t in (p.small, p.ref):
        w = t.new_worker()
        out = []
        for s in sents:
            w.reset_sentence(s)
            w.tokenize()
            out.append([(t_.range_char(), t_.range_byte(), t_.word_idx(), t_.total_cost()) for t_ in w.token_iter()])
        got.append(out)
    assert got[0] == got[1]
    assert p.small.describe()["last_viterbi"] == "k_small_batch" and p.small.last_launch_count() == 1


def test_multi_device_equals_single_device(golden):
    d = adv.make_dictionary("ties", seed=6)
    p = adversarial_pair(d, ignore_space=True)
    dev = vb.SystemDictionaryBuilder.from_readers(d.lex_csv, d.matrix, d.char_def, d.unk_def)
    dev.reset_user_lexicon_from_reader(d.user_csv)
    multi = vb.Tokenizer.new(dev, devices=shard_devices(2)).ignore_space(True).small_batch(64)
    sents = adv.make_sentences(d, 200, seed=2, max_len=60)
    for mode in (None,) + MODES:
        p.set(lambda t: t.output_mode(mode))
        multi.output_mode(mode)
        for batch in ([sents[0]], sents[:3], sents[:64], sents):
            utf8, off = adv.pack(batch)
            a = p.check(utf8, off, mode=mode, route="k_small_batch" if len(batch) <= 64 else "k_viterbi2")
            b = multi.tokenize_batch(utf8=utf8, byte_offsets=off)
            assert_batch_equal(b, a.tok_offsets, a.tokens)
            if mode is not None:
                assert b.text()[1] == a.text()[1]


def _run_on_pty(cmd, data):
    """`cmd` with a pseudo-terminal on stdin (echo off) fed `data`, then end-of-file: its stdout."""
    master, slave = pty.openpty()
    attrs = termios.tcgetattr(slave)
    attrs[3] &= ~termios.ECHO
    termios.tcsetattr(slave, termios.TCSANOW, attrs)
    p = subprocess.Popen(cmd, stdin=slave, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    os.close(slave)
    try:
        os.write(master, data + b"\x04")  # ^D at the start of a line: end of input
        out, err = p.communicate(timeout=120)
    finally:
        os.close(master)
    assert p.returncode == 0, err.decode()
    return out


def test_tokenize_cli_on_a_terminal(golden, tmp_path):
    exe = os.path.join(ROOT, "vibrato_b200", "bin", "tokenize")
    if not os.path.exists(exe):
        pytest.skip("CLIs not built")
    for k, v in golden["resources"].items():
        (tmp_path / k).write_text(v, encoding="utf-8", newline="")
    lines = ["京都東京都京都", "東京 都", "", "kampersanda", "東京県に行く", ""] * 2
    text = ("\n".join(lines) + "\n").encode()
    for mode in MODES:
        for where in ("device", "host"):
            base = [exe, "-i", str(tmp_path), "-u", str(tmp_path / "user.csv"), "-O", mode, "-S", "--format-on", where]
            ref = subprocess.run(base, input=text, capture_output=True, timeout=120)
            assert ref.returncode == 0, ref.stderr.decode()
            one = subprocess.run(base + ["--batch-lines", "1"], input=text, capture_output=True, timeout=120)
            assert one.returncode == 0, one.stderr.decode()
            assert one.stdout == ref.stdout, (mode, where)
            assert _run_on_pty(base, text) == ref.stdout, (mode, where)
