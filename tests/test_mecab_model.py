"""Compact dictionaries from a trained MeCab model: generate_bigram_info (mecab.rs:31-181 of the reference) and the
`mecab_smalldic` CLI (examples/mecab_smalldic/src/main.rs).

CPU: a hand-written model with its three expected files as literals, every error the conversion reports, seeded
random models against the Python restatement in mecab_oracle.py (byte for byte), and the CLI against `compile
--bigram-*`.  GPU: Raw and Dual dictionaries converted from a seeded model tokenise like the oracle, on the whole-batch
and the chunked route, and `mecab_smalldic` -> `tokenize -O detail` prints the oracle's text."""
import os
import subprocess

import numpy as np
import pytest

import adversarial as adv
import mecab_oracle as mo
import vibrato_b200 as vb
from oracle import vibrato_oracle as vo
from vibrato_b200 import synth
from test_dictionary_tools import run, write_sources, zstd_decode

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_FEATURE_DEF = os.path.join(ROOT, "tests", "golden", "feature.def")  # vibrato/src/tests/resources/feature.def

# ---- a hand-written model ----------------------------------------------------------------------------------------
# Left templates (from the left half of each BIGRAM line): B0:%L[0] | B1:%L[0],%L?[2] | B2:%L[1]%R[1] (the %R stays
# literal) | B0:%L[0] again, which shares B0's ids.  Right templates: %R[0] | %R[0],%R?[2] | %R[1]%L[1] | %R?[5].
MINI_FEATURE_DEF = (
    "# comment\n"
    "UNIGRAM U0:%F[0],%F?[1]\n"
    "\n"
    "   BIGRAM B0:%L[0]/%R[0]　\t\n"  # str::trim removes Unicode white space, U+3000 included
    "BIGRAM B1:%L[0],%L?[2]/%R[0],%R?[2]\n"
    "BIGRAM B2:%L[1]%R[1]/%R[1]%L[1]\n"
    "BIGRAM B0:%L[0]/%R?[5]\n"
)
# left features: B0:BOS/EOS=1 B2:*%R[1]=2 | B0:名詞=3 B2:一般%R[1]=4 | B0:助詞=5 B1:助詞,が=6 B2:格助詞%R[1]=7 |
# B0:名詞,固有=8 B2:地名%R[1]=9 | B0:動詞=10 B2:自立%R[1]=11 (id 1 again: it replaces the first row)
MINI_RIGHT_ID_DEF = ("0 BOS/EOS\n"
                     "1 名詞,一般,*\n"
                     "2 助詞,格助詞,が\n"
                     '3 "名詞,固有",地名,*\n'
                     "1 動詞,自立,*")  # no final newline
# right features: BOS/EOS=1 *%L[1]=2 | 名詞=3 一般%L[1]=4 | 助詞=5 格助詞%L[1]=6 x=7
MINI_LEFT_ID_DEF = "0 BOS/EOS,*,*\r\n1 名詞,一般,*,*,*,*\r\n2 助詞,格助詞,*,*,*,x\r\n"
MINI_MODEL_DEF = (
    "version: 102\n"
    "charset: UTF-8\n"
    "cost-factor: 700\n"
    "eval-size: 4\n"
    "\n"
    "0.5\tU0:名詞\n"                        # no '/': skipped
    "1.0\tB0:名詞/助詞\n"                   # 3/5 -700
    "-0.25\tB0:動詞/名詞\n"                 # 10/3 175
    "0.001\tB0:名詞/名詞\n"                 # -0.7 -> 0: skipped
    "-0.0014\tB0:名詞/名詞\n"               # 0.98 -> 0: skipped
    "0.0015\tB0:名詞/名詞\n"                # 3/3 -1
    "-0.9999\tB1:助詞,が/x\n"               # 6/7 699 (toward zero)
    "5000000\tB0:名詞/助詞\n"               # 3/5 saturated to i32::MIN
    "-5000000\tB0:助詞/名詞\n"              # 5/3 saturated to i32::MAX
    "1\tB0:BOS/EOS/名詞\n"                  # "B0:" is no left feature: skipped
    "1\tBOS/EOS/名詞\n"                     # /3 -700
    "2\tB0:助詞/BOS/EOS\n"                  # 5/ -1400
    "1\tBOS/EOS/BOS/EOS\n"                  # / -700
    "1\tB0:未知/名詞\n"                     # unknown left: skipped
    "1\tB0:名詞/未知\n"                     # unknown right: skipped
    "1\tB2:格助詞%R[1]/一般%L[1]\n"         # 7/4 -700
    ".5\tB0:名詞/助詞/extra\n"              # a third piece is ignored: 3/5 -350
    "3.\tB0:動詞/x\n"                       # 10/7 -2100
    "1.0 B0:名詞/助詞\n"                    # a space, not a tab: skipped
    "1.5\n"                                 # skipped
)
MINI_BIGRAM_RIGHT = b"1\t10,*,11,10\n2\t5,6,7,5\n3\t8,*,9,8\n"
MINI_BIGRAM_LEFT = b"1\t3,*,4,*\n2\t5,*,6,7\n"
MINI_BIGRAM_COST = (b"3/5\t-700\n10/3\t175\n3/3\t-1\n6/7\t699\n3/5\t-2147483648\n5/3\t2147483647\n/3\t-700\n"
                    b"5/\t-1400\n/\t-700\n7/4\t-700\n3/5\t-350\n10/7\t-2100\n")


def mini(**over):
    files = {"feature.def": MINI_FEATURE_DEF, "right-id.def": MINI_RIGHT_ID_DEF, "left-id.def": MINI_LEFT_ID_DEF,
             "model.def": MINI_MODEL_DEF}
    files.update(over)
    return files


def convert(files, cost_factor=700, impl=vb.generate_bigram_info):
    return impl(files["feature.def"], files["right-id.def"], files["left-id.def"], files["model.def"], cost_factor)


def test_mini_model_gives_the_expected_files():
    assert convert(mini()) == (MINI_BIGRAM_RIGHT, MINI_BIGRAM_LEFT, MINI_BIGRAM_COST)
    assert convert(mini(), impl=mo.generate_bigram_info) == (MINI_BIGRAM_RIGHT, MINI_BIGRAM_LEFT, MINI_BIGRAM_COST)


def test_golden_feature_def_and_cost_factors():
    """The reference's test feature.def (UNIGRAM lines, four BIGRAM templates, no '?'); cost factors that flip the
    sign, scale to zero and give NaN (0 * inf) leave the ids alone and change only bigram.cost."""
    fd = open(GOLDEN_FEATURE_DEF, encoding="utf-8").read()
    rid = "0 BOS/EOS,*,*,*\n1 名詞,一般,*,*\n2 動詞,自立,*,*,五段\n"
    lid = "0 BOS/EOS\n1 助詞,格助詞,一般,*\n2 名詞,一般,*,*\n"
    model = "1.0\tB1:名詞/助詞\n-2.0\tB2:名詞,一般/名詞,一般\n0.5\tB4:動詞,自立,*,*/BOS/EOS\n1e5\tB1:x/y\n"
    files = {"feature.def": fd, "right-id.def": rid, "left-id.def": lid, "model.def": model}
    right, left, cost = convert(files)
    assert right == b"1\t5,6,7,8\n2\t9,10,11,12\n"
    assert left == b"1\t5,6,7,8\n2\t9,10,11,12\n"
    assert cost == b"5/5\t-700\n6/10\t1400\n12/\t-350\n"  # "1e5": no 'e' in the weight pattern
    for cf, exp in ((-1.0, b"5/5\t1\n6/10\t-2\n"), (0.0, b""), (float("inf"), None), (float("nan"), b"")):
        got = convert(files, cf)
        assert got == convert(files, cf, impl=mo.generate_bigram_info), cf
        assert got[:2] == (right, left)
        if exp is not None:
            assert got[2] == exp, cf
    assert convert(files, float("inf"))[2] == b"5/5\t-2147483648\n6/10\t2147483647\n12/\t-2147483648\n"


ERRORS = [
    # (what, files, VibratoError kind, message fragment)
    ("right id 0 is not BOS/EOS", mini(**{"right-id.def": "0 名詞\n1 名詞,一般,*\n"}), "InvalidFormat",
     "right_id_def_rdr: ID 0 must be BOS/EOS"),
    ("left id 0 is not BOS/EOS", mini(**{"left-id.def": "0 BOS/EOS2\n1 名詞\n"}), "InvalidFormat",
     "left_id_def_rdr: ID 0 must be BOS/EOS"),
    ("blank id line", mini(**{"right-id.def": "0 BOS/EOS\n\n1 名詞\n"}), "InvalidFormat",
     "right_id_def_rdr: each line must be a pair of an ID and features"),
    ("id without a space", mini(**{"left-id.def": "0 BOS/EOS\n1名詞\n"}), "InvalidFormat",
     "left_id_def_rdr: each line must be a pair"),
    ("id not a number", mini(**{"left-id.def": "0 BOS/EOS\nx 名詞\n"}), "InvalidFormat", "left_id_def_rdr"),
    ("space before the id", mini(**{"right-id.def": " 0 BOS/EOS\n"}), "InvalidFormat", "right_id_def_rdr"),
    ("tab instead of a space", mini(**{"right-id.def": "0\tBOS/EOS\n"}), "InvalidFormat", "right_id_def_rdr"),
    ("id past usize", mini(**{"right-id.def": "0 BOS/EOS\n18446744073709551616 名詞\n"}), "ParseInt", ""),
    ("undefined right-id", mini(**{"right-id.def": "0 BOS/EOS\n1 名詞\n3 名詞\n"}), "InvalidFormat",
     "right_id_def_rdr: feature ID 2 is undefined"),
    ("undefined left-id", mini(**{"left-id.def": "0 BOS/EOS\n2 名詞\n4 名詞\n"}), "InvalidFormat",
     "left_id_def_rdr: feature ID 1 is undefined"),
    ("two slashes in BIGRAM", mini(**{"feature.def": "BIGRAM a/b/c\n"}), "InvalidFormat",
     "feature.def: Invalid bigram template"),
    ("no slash in BIGRAM", mini(**{"feature.def": "BIGRAM %L[0]\n"}), "InvalidFormat", "Invalid bigram template"),
    ("unknown feature.def line", mini(**{"feature.def": "TRIGRAM x\n"}), "InvalidFormat", "feature: "),
    ("UNIGRAM without its space", mini(**{"feature.def": "UNIGRAM\n"}), "InvalidFormat", "feature: "),
    ("lower-case keyword", mini(**{"feature.def": "bigram %L[0]/%R[0]\n"}), "InvalidFormat", "feature: "),
    ("template index past usize", mini(**{"feature.def": "BIGRAM %L[18446744073709551616]/%R[0]\n"}), "ParseInt", ""),
    ("invalid UTF-8", mini(**{"model.def": b"1\tB0:\xff/x\n"}), "StdIo", "valid UTF-8"),
]
ERRORS += [(f"weight {w!r}", mini(**{"model.def": MINI_MODEL_DEF + f"{w}\tB0:名詞/助詞\n"}), "ParseFloat", "")
           for w in ("-", ".", "-.", "1.2.3", "1-2", "--1", "1.-")]


@pytest.mark.parametrize("what,files,kind,msg", ERRORS, ids=[e[0] for e in ERRORS])
def test_conversion_errors(what, files, kind, msg):
    with pytest.raises(vb.VibratoError) as ei:
        convert(files)
    assert ei.value.kind == kind and msg in str(ei.value), str(ei.value)
    assert ei.value.code == {"InvalidFormat": 2, "ParseInt": 4, "StdIo": 7, "ParseFloat": 10}[kind]
    with pytest.raises(mo.MecabOracleError) as eo:
        convert(files, impl=mo.generate_bigram_info)
    assert eo.value.kind == kind


def test_highest_id_is_dropped_without_id_0():
    """1..len(map) are written: with no id 0 the map is one short and its highest id is silently left out, as in the
    reference; an id above the others is then allowed to be anything."""
    for rid in ("1 名詞,一般,*\n2 助詞,格助詞,が\n", "2 助詞,格助詞,が\n1 名詞,一般,*\n900 動詞\n"):
        right, left, cost = convert(mini(**{"right-id.def": rid}))
        assert right.decode().splitlines() == (["1\t1,*,2,1"] if rid.startswith("1") else ["1\t4,*,5,4", "2\t1,2,3,1"])
        assert (right, left, cost) == convert(mini(**{"right-id.def": rid}), impl=mo.generate_bigram_info)
    right, left, _ = convert(mini(**{"left-id.def": "1 名詞\n"}))
    assert left == b""


def test_empty_and_missing_sources():
    assert convert(mini(**{"feature.def": "", "right-id.def": "", "left-id.def": "", "model.def": ""})) == (b"", b"", b"")
    right, left, cost = convert(mini(**{"feature.def": "# nothing\n"}))
    assert right == b"1\t\n2\t\n3\t\n" and left == b"1\t\n2\t\n" and cost == b"/\t-700\n"  # BOS/EOS/BOS/EOS


def mutated_model(seed, n_templates):
    """A synthetic unidic-shaped model, plus what a real one may hold: templates whose left half holds a literal %R[..]
    and a missing optional index, a repeated id (it replaces the first), CRLF line ends, a final line without "\\n"."""
    rng = np.random.default_rng(seed)
    m = synth.make_mecab_model(60 + seed, 50 + 2 * seed, n_templates=n_templates, n_model_lines=4000, seed=seed)
    m["feature.def"] += "BIGRAM M0:%L?[1]%R[2]x/%R[0]%L?[3]\nBIGRAM M1:%L?[12],%L[2]/%R?[12],%R[2]\n"
    for key in ("left-id.def", "right-id.def"):
        lines = m[key].splitlines()
        k = int(rng.integers(1, len(lines)))
        lines.append(f"{k} " + lines[int(rng.integers(1, len(lines)))].split(" ", 1)[1])
        lines.append('1 名詞,細0,*,*,*,*,"語1,2",*,"x""y"')  # quoted fields, one holding a comma
        m[key] = "\n".join(lines)
    if seed % 2:
        m["model.def"] = m["model.def"].replace("\n", "\r\n")
    return m


@pytest.mark.parametrize("seed,n_templates", [(1, 9), (2, 12), (3, 16), (4, 24)])
def test_random_models_match_the_oracle(seed, n_templates):
    m = mutated_model(seed, n_templates)
    assert m["feature.def"].count("?") >= 9 and '"' in m["right-id.def"] and '"' in m["left-id.def"]
    for cf in (700.0, 1.0, 0.37, -3.0, 1e9):
        got = convert(m, cf)
        assert got == convert(m, cf, impl=mo.generate_bigram_info), cf
        assert got[2], cf
    right, left, cost = convert(m)
    assert len(right.splitlines()) == 50 + 2 * seed - 1 and len(left.splitlines()) == 60 + seed - 1
    assert b"*" in right and b"\t/" not in cost
    assert any(ln.startswith(b"/") for ln in cost.splitlines()) and any(b"/\t" in ln for ln in cost.splitlines())


def test_cpp_mirror_matches_python(tmp_path):
    """vibrato_b200.hpp's mecab::generate_bigram_info, through a small program."""
    import shutil
    cxx = os.environ.get("CXX") or shutil.which("c++") or shutil.which("g++")
    so_dir = os.path.join(ROOT, "vibrato_b200")
    if not cxx or not os.path.exists(os.path.join(so_dir, "libvibrato_b200.so")):
        pytest.skip("no C++ compiler or library")
    (tmp_path / "m.cpp").write_text(r"""
#include <fstream>
#include <iostream>
#include <sstream>
#include "vibrato_b200.hpp"
static std::string slurp(const char* p) { std::ifstream f(p, std::ios::binary); std::stringstream s; s << f.rdbuf(); return s.str(); }
int main(int, char** argv) {
    try {
        auto b = vibrato_b200::mecab::generate_bigram_info(slurp(argv[1]), slurp(argv[2]), slurp(argv[3]), slurp(argv[4]), 700);
        std::cout << b.right << "=\n" << b.left << "=\n" << b.cost;
    } catch (const vibrato_b200::VibratoError& e) {
        std::cout << "error " << e.code << "\n";
    }
}
""")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(so_dir, "cpp"), str(tmp_path / "m.cpp"), "-o",
                           str(tmp_path / "m"), "-L", so_dir, "-lvibrato_b200", f"-Wl,-rpath,{so_dir}"])
    for files in (mini(), mini(**{"model.def": "1.2.3\tx/y\n"})):
        src = write_sources(tmp_path / "src", files)
        out = subprocess.run([str(tmp_path / "m")] + [str(src / k) for k in ("feature.def", "right-id.def",
                                                                            "left-id.def", "model.def")],
                             capture_output=True, check=True).stdout
        if files["model.def"] == MINI_MODEL_DEF:
            assert out == MINI_BIGRAM_RIGHT + b"=\n" + MINI_BIGRAM_LEFT + b"=\n" + MINI_BIGRAM_COST
        else:
            assert out == b"error 10\n"


# ---- the CLI -------------------------------------------------------------------------------------------------------

def smalldic_args(src, out, dual):
    return (["-l", f"{src}/lex.csv", "-u", f"{src}/unk.def", "-c", f"{src}/char.def", "-f", f"{src}/feature.def",
             "-a", f"{src}/right-id.def", "-b", f"{src}/left-id.def", "-m", f"{src}/model.def", "-r", "700", "-o", out]
            + (["--dual-connector"] if dual else []))


@pytest.mark.parametrize("dual", [False, True])
def test_mecab_smalldic_writes_what_compile_writes(tmp_path, dual):
    sd = synth.make_dictionary("synth-tiny")
    files = synth.make_mecab_model(sd.num_left, sd.num_right, n_templates=12, n_model_lines=6000, seed=7)
    right, left, cost = convert(files)
    files.update({"lex.csv": sd.lex_csv, "char.def": sd.char_def, "unk.def": sd.unk_def, "bigram.right": right,
                  "bigram.left": left, "bigram.cost": cost})
    src = write_sources(tmp_path / "src", files)
    out = tmp_path / "small.dic.zst"
    p = run("mecab_smalldic", *smalldic_args(src, out, dual))
    assert p.returncode == 0, p.stderr.decode()
    err = p.stderr.decode().splitlines()
    assert len(err) == 3 and err[0] == "Compiling the system dictionary..."
    assert err[1].endswith(" seconds") and float(err[1].split()[0]) >= 0
    assert err[2] == f'Writing the system dictionary in zstd...: "{out}"'
    p = run("compile", "-l", f"{src}/lex.csv", "-u", f"{src}/unk.def", "-c", f"{src}/char.def", "-o",
            tmp_path / "compiled.dic.zst", "--bigram-right-in", f"{src}/bigram.right", "--bigram-left-in",
            f"{src}/bigram.left", "--bigram-cost-in", f"{src}/bigram.cost", *(["--dual-connector"] if dual else []))
    assert p.returncode == 0, p.stderr.decode()
    assert zstd_decode(out) == zstd_decode(tmp_path / "compiled.dic.zst")


def test_mecab_smalldic_errors(tmp_path):
    sd = synth.make_dictionary("synth-tiny")
    files = synth.make_mecab_model(sd.num_left, sd.num_right, n_templates=12, n_model_lines=100, seed=8)
    files.update({"lex.csv": sd.lex_csv, "char.def": sd.char_def, "unk.def": sd.unk_def})
    src = write_sources(tmp_path / "src", files)
    out = tmp_path / "small.dic.zst"
    args = smalldic_args(src, out, False)
    r = args.index("-r")
    for bad in (args[:r] + args[r + 2:], args[:r + 1] + ["seven"] + args[r + 2:], args[:-2], args + ["-x"]):
        assert run("mecab_smalldic", *bad).returncode == 2
    write_sources(src, {"model.def": files["model.def"] + "1.2.3\tB00:x/y\n"})
    p = run("mecab_smalldic", *args)
    assert p.returncode == 1 and b"Error: " in p.stderr and not out.exists()
    write_sources(src, {"model.def": files["model.def"]})
    (src / "left-id.def").unlink()
    p = run("mecab_smalldic", *args)
    assert p.returncode == 1 and b"Error: " in p.stderr and not out.exists()


# ---- GPU: tokenisation with converted dictionaries ----------------------------------------------------------------

def reid(csv_text, left_map, right_map):
    """lex.csv / unk.def rows with their left and right ids (columns 1, 2) renamed through the maps."""
    rows = []
    for row in csv_text.splitlines():
        f = row.split(",")
        f[1], f[2] = str(left_map[int(f[1])]), str(right_map[int(f[2])])
        rows.append(",".join(f))
    return "\n".join(rows) + "\n"


NUM_LEFT, NUM_RIGHT = 48, 41


def converted_sources(source):
    """(lex.csv, char.def, unk.def, sentences) with the ids 1..9 of the source spread over the model's ids."""
    rng = np.random.default_rng(11)
    lmap = dict(zip(range(1, 10), (rng.choice(NUM_LEFT - 1, 9, replace=False) + 1).tolist()))
    rmap = dict(zip(range(1, 10), (rng.choice(NUM_RIGHT - 1, 9, replace=False) + 1).tolist()))
    if source == "fixture":
        import json
        with open(os.path.join(ROOT, "tests", "golden", "vibrato_fixture.json"), encoding="utf-8") as f:
            g = json.load(f)
        r = g["resources"]
        d = adv.make_dictionary("ties", seed=3)
        sents = [c["input"] for c in g["tokenizer_cases"]] + ["東京に行った。", "", "京都東京都京都"]
        sents += adv.make_sentences(d, 600, seed=5)
        return reid(r["lex.csv"], lmap, rmap), r["char.def"], reid(r["unk.def"], lmap, rmap), sents
    d = adv.make_dictionary(source, seed=4)
    return reid(d.lex_csv, lmap, rmap), d.char_def, reid(d.unk_def, lmap, rmap), adv.make_sentences(d, 1500, seed=6)


def model_and_bigram(n_templates):
    m = synth.make_mecab_model(NUM_LEFT, NUM_RIGHT, n_templates=n_templates, n_model_lines=8000, seed=21)
    bigram = convert(m)
    assert bigram == convert(m, impl=mo.generate_bigram_info)
    return m, bigram


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["fixture", "ties", "extreme"])
@pytest.mark.parametrize("dual", [False, True])
def test_converted_dictionary_tokenizes_like_the_oracle(source, dual):
    lex, char_def, unk, sents = converted_sources(source)
    _, (right, left, cost) = model_and_bigram(12)
    d = vb.SystemDictionaryBuilder.from_readers_with_bigram_info(lex, right, left, cost, char_def, unk,
                                                                 dual_connector=dual)
    od = vo.OracleDictionary(lex, (right, left, cost), char_def, unk, dual_connector=dual)
    utf8, off = adv.pack(sents)
    tok_off, toks, cnt = od.tokenize_batch(utf8, off, False, n_threads=8, want_counters=True)
    etext = vo.format_batch(od, utf8, off, tok_off, toks, "detail")
    tok = vb.Tokenizer.new(d)
    for chunk in (0, 256):  # the whole batch, and the chunked host pipeline
        tok.set_option("chunk_sentences", chunk)
        tok.set_counting(True)
        res = tok.tokenize_batch(utf8=utf8, byte_offsets=off)
        np.testing.assert_array_equal(res.tok_offsets, tok_off)
        for name in vb.TOKEN_DTYPE.names:
            np.testing.assert_array_equal(res.tokens[name], toks[name], err_msg=name)
        np.testing.assert_array_equal(tok.last_counters(), cnt)
        tok.set_counting(False)
        res = tok.output_mode("detail").tokenize_batch(utf8=utf8, byte_offsets=off)
        toff, text = res.text()
        np.testing.assert_array_equal(toff, etext[0])
        assert text == etext[1], chunk
        tok.output_mode(None)


@pytest.mark.gpu
@pytest.mark.parametrize("dual", [False, True])
def test_mecab_smalldic_then_tokenize_detail(tmp_path, dual):
    lex, char_def, unk, sents = converted_sources("fixture")
    m, bigram = model_and_bigram(10)
    src = write_sources(tmp_path / "src", dict(m, **{"lex.csv": lex, "char.def": char_def, "unk.def": unk}))
    out = tmp_path / "small.dic.zst"
    p = run("mecab_smalldic", *smalldic_args(src, out, dual))
    assert p.returncode == 0, p.stderr.decode()
    sents = [s for s in sents if "\n" not in s and "\r" not in s]
    p = run("tokenize", "-i", out, "-O", "detail", stdin=("\n".join(sents) + "\n").encode())
    assert p.returncode == 0, p.stderr.decode()
    od = vo.OracleDictionary(lex, bigram, char_def, unk, dual_connector=dual)
    utf8, off = adv.pack(sents)
    tok_off, toks = od.tokenize_batch(utf8, off, False, n_threads=8)[:2]
    assert p.stdout == vo.format_batch(od, utf8, off, tok_off, toks, "detail")[1]
