"""The dictionary tool chain: Dictionary.write_zstd_file and the `compile` / `reorder` / `map` CLIs
(compile/src/main.rs, map/src/reorder.rs, map/src/main.rs of the reference).

CPU: `compile` and `map` against the Python builders (their output decompressed by a decoder of its own), their
argument and input errors, the `.lmap` / `.rmap` naming and the probability text of `reorder` through a small program
built on the CLIs' shared header.  GPU: `reorder` against the oracle's connection-id counts, and the whole flow
compile -> reorder -> map -> tokenize."""
import ctypes as C
import math
import os
import shutil
import subprocess
from decimal import Decimal

import numpy as np
import pytest

import vibrato_b200 as vb
from vibrato_b200 import synth
from oracle import vibrato_oracle as vo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "vibrato_b200", "bin")
SOURCES = ("lex.csv", "matrix.def", "char.def", "unk.def")


def tool(name):
    exe = os.path.join(BIN, name)
    if not os.path.exists(exe):
        pytest.skip("CLIs not built")
    return exe


def run(name, *args, stdin=b"", cwd=None):
    return subprocess.run([tool(name)] + [str(a) for a in args], input=stdin, capture_output=True, timeout=600, cwd=cwd)


def zstd_decode(path):
    """One zstd frame -> bytes, through libzstd's one-shot API (not the library's streaming decoder)."""
    try:
        z = C.CDLL("libzstd.so.1")
    except OSError:
        pytest.skip("libzstd.so.1 not present")
    z.ZSTD_getFrameContentSize.restype = C.c_ulonglong
    z.ZSTD_getFrameContentSize.argtypes = [C.c_void_p, C.c_size_t]
    z.ZSTD_decompress.restype = C.c_size_t
    z.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    z.ZSTD_isError.restype = C.c_uint
    z.ZSTD_isError.argtypes = [C.c_size_t]
    comp = open(path, "rb").read()
    n = z.ZSTD_getFrameContentSize(comp, len(comp))
    assert n < (1 << 62), "the frame header must carry the content size"
    out = C.create_string_buffer(max(n, 1))
    got = z.ZSTD_decompress(out, n, comp, len(comp))
    assert not z.ZSTD_isError(got) and got == n
    return out.raw[:n]


def write_sources(dst, files):
    os.makedirs(dst, exist_ok=True)
    for k, v in files.items():
        with open(os.path.join(dst, k), "wb") as f:
            f.write(v.encode("utf-8") if isinstance(v, str) else bytes(v))
    return dst


def fixture_sources(golden):
    return {k: golden["resources"][k] for k in SOURCES}


def synth_sources(name):
    sd = synth.make_dictionary(name)
    return sd, {"lex.csv": sd.lex_csv, "matrix.def": sd.matrix_def(), "char.def": sd.char_def, "unk.def": sd.unk_def}


def compile_args(src, out):
    return ["-l", f"{src}/lex.csv", "-m", f"{src}/matrix.def", "-u", f"{src}/unk.def", "-c", f"{src}/char.def",
            "-o", out]


def python_dict(files):
    return vb.SystemDictionaryBuilder.from_readers(files["lex.csv"], files["matrix.def"], files["char.def"],
                                                   files["unk.def"])


# ---- Rust's formatting, restated ------------------------------------------------------------------------------------

def rust_f64(x):
    """`{}` of an f64: the shortest digits that round-trip (what repr prints), positional, never an exponent."""
    if math.isnan(x):
        return "NaN"
    s = format(Decimal(repr(x)), "f")
    return s.rstrip("0").rstrip(".") if "." in s else s


def mapping_text(counts):
    """ConnIdCounter::compute_probs (mapper.rs:108-146) for one side, written as reorder.rs:50-52 writes it."""
    total = float(sum(int(c) for c in counts))
    probs = [(i, float(c) / total if total else float("nan")) for i, c in enumerate(counts)][1:]
    if total:
        probs.sort(key=lambda t: (-t[1], t[0]))  # without NaN: no pair is incomparable
    return "".join(f"{i}\t{rust_f64(p)}\n" for i, p in probs)


# ---- CPU: write_zstd_file, compile, map ------------------------------------------------------------------------------

def test_write_zstd_file_round_trips_and_reports_io_errors(golden, tmp_path):
    d = python_dict(fixture_sources(golden)).reset_user_lexicon_from_reader(golden["resources"]["user.csv"])
    stream = d.write()
    for level in (19, 3):
        path = tmp_path / f"system{level}.dic.zst"
        assert d.write_zstd_file(path, level) is d
        assert zstd_decode(path) == stream
        assert vb.Dictionary.from_zstd_file(path).write() == stream
    for bad in (tmp_path / "no-such-dir" / "x.dic.zst", tmp_path):
        with pytest.raises(vb.VibratoError) as ei:
            d.write_zstd_file(bad)
        assert ei.value.kind == "StdIo" and ei.value.code == 7
    assert not (tmp_path / "no-such-dir").exists()


@pytest.mark.parametrize("connector", ["matrix", "raw", "dual"])
def test_compile_writes_what_the_python_builder_builds(golden, tmp_path, connector):
    build = vb.SystemDictionaryBuilder
    if connector == "matrix":
        files = fixture_sources(golden)
        src = write_sources(tmp_path / "src", files)
        args = compile_args(src, tmp_path / "system.dic.zst")
        d = python_dict(files)
    else:
        sd, files = synth_sources("synth-tiny")
        right, left, cost = synth.make_bigram_files(sd, n_templates=12)
        files.update({"bigram.right": right, "bigram.left": left, "bigram.cost": cost})
        src = write_sources(tmp_path / "src", files)
        # -m absent: the bigram files decide; --dual-connector picks the Dual connector (compile/src/main.rs:69-82)
        args = ["-l", f"{src}/lex.csv", "-u", f"{src}/unk.def", "-c", f"{src}/char.def", "-o", tmp_path / "system.dic.zst",
                "--bigram-right-in", f"{src}/bigram.right", "--bigram-left-in", f"{src}/bigram.left",
                "--bigram-cost-in", f"{src}/bigram.cost"] + (["--dual-connector"] if connector == "dual" else [])
        d = build.from_readers_with_bigram_info(sd.lex_csv, right, left, cost, sd.char_def, sd.unk_def,
                                                dual_connector=connector == "dual")
    p = run("compile", *args)
    assert p.returncode == 0, p.stderr.decode()
    err = p.stderr.decode().splitlines()
    assert err[0] == "Compiling the system dictionary..." and err[1].endswith(" seconds")
    assert err[2] == f'Writing the system dictionary in zstd...: "{tmp_path / "system.dic.zst"}"'
    stream = d.write()
    assert zstd_decode(tmp_path / "system.dic.zst") == stream
    assert vb.Dictionary.from_zstd_file(tmp_path / "system.dic.zst").write() == stream


def test_compile_argument_and_source_errors(golden, tmp_path):
    files = fixture_sources(golden)
    src = write_sources(tmp_path / "src", files)
    out = tmp_path / "system.dic.zst"
    no_connector = ["-l", f"{src}/lex.csv", "-u", f"{src}/unk.def", "-c", f"{src}/char.def", "-o", out]
    for extra in ([], ["--bigram-right-in", f"{src}/lex.csv", "--bigram-left-in", f"{src}/lex.csv"]):
        p = run("compile", *(no_connector + extra))
        assert p.returncode == 2
        assert b"At least one of --matrin-in or --bigram-{right,left,cost}-in must be specified." in p.stderr
    assert run("compile", *compile_args(src, out)[:-2]).returncode == 2  # no -o
    assert run("compile", "--no-such-flag").returncode == 2
    assert not out.exists()
    bad = write_sources(tmp_path / "bad", dict(files, **{"lex.csv": "短い,1,x,100,形容詞\n" + files["lex.csv"]}))
    p = run("compile", *compile_args(bad, out))
    assert p.returncode == 1 and b"Error: " in p.stderr and not out.exists()
    p = run("compile", *compile_args(tmp_path / "missing", out))
    assert p.returncode == 1 and b"Error: " in p.stderr and not out.exists()


def fixture_dic(golden, tmp_path):
    files = fixture_sources(golden)
    path = tmp_path / "system.dic.zst"
    python_dict(files).write_zstd_file(path, 3)
    return files, path


def test_map_applies_the_mapping_files(golden, tmp_path):
    files, dic = fixture_dic(golden, tmp_path)
    shape = python_dict(files).shape()
    rng = np.random.default_rng(5)
    lmap = (rng.permutation(shape["num_left"] - 1) + 1).tolist()
    rmap = (rng.permutation(shape["num_right"] - 1) + 1).tolist()
    # the first tab-separated column counts; "+5" is a u16 to Rust, and "\r\n" ends a line as "\n" does
    ltext = "".join(f"{'+' if k == 3 else ''}{i}\t{0.5 / (k + 1)}\tanything\n" for k, i in enumerate(lmap))
    rtext = "".join(f"{i}\tx" + ("\r\n" if k == 1 else "\n") for k, i in enumerate(rmap))
    (tmp_path / "reordered.lmap").write_text(ltext)
    (tmp_path / "reordered.rmap").write_bytes(rtext.encode())
    out = tmp_path / "mapped.dic.zst"
    p = run("map", "-i", dic, "-m", tmp_path / "reordered", "-o", out)
    assert p.returncode == 0, p.stderr.decode()
    assert p.stderr.decode() == ("Loading the dictionary...\nLoading and doing the mapping...\n"
                                 f'Writing the mapped system dictionary...: "{out}"\n')
    assert zstd_decode(out) == python_dict(files).map_connection_ids_from_iter(lmap, rmap).write()


def test_map_rejects_bad_mapping_files(golden, tmp_path):
    files, dic = fixture_dic(golden, tmp_path)
    shape = python_dict(files).shape()
    good_l = [str(i) for i in range(1, shape["num_left"])]
    good_r = "".join(f"{i}\n" for i in range(1, shape["num_right"]))
    cases = {
        "id 0": ["0"] + good_l[1:],
        "duplicate": good_l[:-1] + [good_l[0]],
        "out of range": good_l[:-1] + [str(shape["num_left"])],
        "65536": good_l[:-1] + ["65536"],
        "empty line": good_l[:-1] + [""],
        "leading space": good_l[:-1] + [" " + good_l[-1]],
        "minus": good_l[:-1] + ["-" + good_l[-1]],
        "lone plus": good_l[:-1] + ["+"],
    }
    out = tmp_path / "mapped.dic.zst"
    for what, lines in cases.items():
        (tmp_path / "m.lmap").write_text("".join(f"{x}\n" for x in lines))
        (tmp_path / "m.rmap").write_text(good_r)
        p = run("map", "-i", dic, "-m", tmp_path / "m", "-o", out)
        assert p.returncode == 1 and b"Error: " in p.stderr, what
        assert not out.exists(), what
    (tmp_path / "m.lmap").write_text("".join(f"{x}\n" for x in good_l))
    (tmp_path / "m.rmap").unlink()
    p = run("map", "-i", dic, "-m", tmp_path / "m", "-o", out)
    assert p.returncode == 1 and not out.exists()
    assert run("map", "-i", dic, "-m", tmp_path / "m").returncode == 2
    (tmp_path / "m.rmap").write_text(good_r)
    assert run("map", "-i", dic, "-m", tmp_path / "m", "-o", out).returncode == 0 and out.exists()


SET_EXTENSION = [("reordered", "reordered.lmap"), ("out/v1.x", "out/v1.lmap"), ("a.b.c", "a.b.lmap"),
                 (".hidden", ".hidden.lmap")]


def test_map_finds_mapping_files_by_set_extension(golden, tmp_path):
    files, dic = fixture_dic(golden, tmp_path)
    shape = python_dict(files).shape()
    (tmp_path / "out").mkdir()
    for arg, lmap in SET_EXTENSION:
        rmap = lmap[:-len("lmap")] + "rmap"
        (tmp_path / lmap).write_text("".join(f"{i}\n" for i in range(1, shape["num_left"])))
        (tmp_path / rmap).write_text("".join(f"{i}\n" for i in range(1, shape["num_right"])))
        p = run("map", "-i", dic, "-m", arg, "-o", "mapped.dic.zst", cwd=tmp_path)
        assert p.returncode == 0, (arg, p.stderr.decode())
        (tmp_path / lmap).unlink()
        (tmp_path / rmap).unlink()
        (tmp_path / "mapped.dic.zst").unlink()


def test_reorder_arguments_before_the_gpu(golden, tmp_path):
    _, dic = fixture_dic(golden, tmp_path)
    for args in ([], ["-i", dic], ["-o", tmp_path / "m"], ["-i", dic, "-o", tmp_path / "m", "--batch-lines", "0"],
                 ["-i", dic, "-o", tmp_path / "m", "--batch-lines", "many"],
                 ["-i", dic, "-o", tmp_path / "m", "--devices", "zero"], ["-i", dic, "-o", tmp_path / "m", "-x"]):
        assert run("reorder", *args, stdin=b"a\n").returncode == 2, args
    p = run("reorder", "-i", tmp_path / "missing.dic.zst", "-o", tmp_path / "m", stdin=b"a\n")
    assert p.returncode == 1 and b"Error: " in p.stderr
    assert not list(tmp_path.glob("m.*"))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    """A program over the CLIs' shared header: rust_f64, the mapping text of reorder, set_extension, Rust's {:?}."""
    cxx = os.environ.get("CXX") or shutil.which("c++") or shutil.which("g++")
    if not cxx:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("harness")
    (d / "h.cpp").write_text(r"""
#include <cstdlib>
#include <iostream>
#include "cli_common.hpp"
int main(int argc, char** argv) {
    const std::string mode = argv[1];
    std::string s;
    if (mode == "f") while (std::cin >> s) std::cout << cli::rust_f64(std::strtod(s.c_str(), nullptr)) << "\n";
    if (mode == "e") while (std::getline(std::cin, s)) std::cout << cli::set_extension(s, "lmap") << "\n";
    if (mode == "d") while (std::getline(std::cin, s)) std::cout << cli::rust_debug_path(s) << "\n";
    if (mode == "p") {
        std::vector<uint64_t> counts;
        while (std::cin >> s) counts.push_back(std::stoull(s));
        std::cout << cli::mapping_text(vibrato_b200::compute_connid_probs(counts));
    }
}
""")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "vibrato_b200", "cpp"), str(d / "h.cpp"),
                           "-o", str(d / "h")])

    def call(mode, text):
        return subprocess.run([str(d / "h"), mode], input=text.encode(), capture_output=True, check=True).stdout.decode()
    return call


def test_probability_text_is_rusts(harness):
    values = [0.5, 0.1, 1 / 3, 1e-7, 1.0, 0.0, float("nan")]
    assert harness("f", "\n".join(map(repr, values))).split() == ["0.5", "0.1", "0.3333333333333333", "0.0000001", "1",
                                                                  "0", "NaN"]
    rng = np.random.default_rng(11)
    xs = [float(a) / float(b) for a, b in zip(rng.integers(0, 10**9, 400), rng.integers(1, 10**12, 400))]
    xs += [float(x) for x in rng.random(100) * 10.0 ** rng.integers(-20, 6, 100)]
    assert harness("f", "\n".join(map(repr, xs))).split() == [rust_f64(x) for x in xs]
    for n, hi in ((50, 5), (300, 10**6), (1, 3), (40, 1)):
        counts = rng.integers(0, hi, n).tolist()
        assert harness("p", " ".join(map(str, counts))) == mapping_text(counts), (n, hi)
    zeros = [0] * 20  # an empty corpus: every probability NaN, in id order
    assert harness("p", " ".join(map(str, zeros))) == "".join(f"{i}\tNaN\n" for i in range(1, 20))


def test_set_extension_and_debug_paths_follow_rust(harness):
    cases = SET_EXTENSION + [("out/", "out.lmap"), ("a/.", "a.lmap"), ("x/a.", "x/a.lmap"), ("..b", "..lmap"),
                             ("dir/.hidden", "dir/.hidden.lmap"), ("", ""), ("/", "/"), (".", "."), ("..", ".."),
                             ("a/..", "a/.."), ("./", "./"), ("/.", "/.")]
    assert harness("e", "".join(f"{a}\n" for a, _ in cases)).split("\n")[:-1] == [b for _, b in cases]
    assert harness("d", 'plain\na"b\\c\td\n').splitlines() == ['"plain"', '"a\\"b\\\\c\\td"']


# ---- GPU: reorder, and the whole flow --------------------------------------------------------------------------------

def gpu_count():
    import torch
    return torch.cuda.device_count()


def substituted(lines):
    """What reorder counts: every empty line stands for the last non-empty line before it."""
    out, last = [], None
    for ln in lines:
        last = ln if ln else last
        out.append(last)
    return out


def expected_maps(od, lines):
    utf8, off = vb.Tokenizer.pack(substituted(lines))
    lid, rid = od.connid_counts(utf8, off, n_threads=8)
    return mapping_text(lid), mapping_text(rid)


def corpus_lines(sd, n, seed):
    utf8, off = synth.make_corpus(sd, n, seed=seed, log_uniform=(1, 80), unk_frac=0.1)
    b = bytes(utf8)
    return [b[int(off[i]):int(off[i + 1])].decode("utf-8") for i in range(n)]


@pytest.mark.gpu
def test_reorder_counts_like_the_reference(tmp_path):
    sd, files = synth_sources("synth-small")
    dic = tmp_path / "system.dic.zst"
    python_dict(files).write_zstd_file(dic, 3)
    od = vo.OracleDictionary(sd.lex_csv, sd.matrix, sd.char_def, sd.unk_def)
    lines = corpus_lines(sd, 3000, seed=41)
    rng = np.random.default_rng(42)
    for i in sorted(rng.choice(np.arange(1, 3000), 60, replace=False).tolist()):
        lines[i] = ""
    lines[500] = lines[1000] = lines[1001] = ""  # the first line of the second batch, and a run of two
    lines.insert(2000, "")
    stdin = ("\n".join(lines) + "\n").encode()
    exp_l, exp_r = expected_maps(od, lines)
    arms = [[], ["--devices", "0"]] + ([["--devices", "0,1"]] if gpu_count() >= 2 else [])
    for extra in arms:
        out = tmp_path / f"m{len(extra)}"
        p = run("reorder", "-i", dic, "-o", out, "--batch-lines", 500, *extra, stdin=stdin)
        assert p.returncode == 0, p.stderr.decode()
        assert p.stdout.decode() == f'Wrote "{out}.lmap"\nWrote "{out}.rmap"\n'
        assert p.stderr.decode() == ("Loading the dictionary...\nReordering connection id mappings...\n"
                                     "Writing connection id mappings...\n")
        assert (tmp_path / f"m{len(extra)}.lmap").read_text() == exp_l, extra
        assert (tmp_path / f"m{len(extra)}.rmap").read_text() == exp_r, extra


@pytest.mark.gpu
def test_reorder_edge_inputs(golden, tmp_path):
    files, dic = fixture_dic(golden, tmp_path)
    shape = python_dict(files).shape()
    for stdin in (b"\n\xe4\xba\xac\xe9\x83\xbd\n", "京都\n東京\n".encode() + b"\xff\xfe\n" + "京都\n".encode()):
        p = run("reorder", "-i", dic, "-o", tmp_path / "m", stdin=stdin)
        assert p.returncode != 0 and b"Error: " in p.stderr and p.stdout == b""
        assert not list(tmp_path.glob("m.*"))
    p = run("reorder", "-i", dic, "-o", tmp_path / "m", stdin=b"")
    assert p.returncode == 0, p.stderr.decode()
    assert (tmp_path / "m.lmap").read_text() == "".join(f"{i}\tNaN\n" for i in range(1, shape["num_left"]))
    assert (tmp_path / "m.rmap").read_text() == "".join(f"{i}\tNaN\n" for i in range(1, shape["num_right"]))
    (tmp_path / "out").mkdir()
    for arg, lmap in SET_EXTENSION:
        p = run("reorder", "-i", dic, "-o", arg, stdin="京都東京都\n".encode(), cwd=tmp_path)
        rmap = lmap[:-len("lmap")] + "rmap"
        assert p.returncode == 0 and p.stdout.decode() == f'Wrote "{lmap}"\nWrote "{rmap}"\n', arg
        assert (tmp_path / lmap).exists() and (tmp_path / rmap).exists()


def detail_ids(line):
    f = dict(x.split("=", 1) for x in line.split("\t") if "=" in x)
    return int(f["left_id"]), int(f["right_id"])


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["fixture", "synth-small"])
def test_compile_reorder_map_tokenize(golden, tmp_path, source):
    if source == "fixture":
        files = fixture_sources(golden)
        lines = [c["input"] for c in golden["tokenizer_cases"]] + ["東京に行った。", "", "京都東京都京都"]
    else:
        sd, files = synth_sources("synth-small")
        lines = corpus_lines(sd, 2000, seed=43)
    lines = [ln for ln in lines if "\n" not in ln and "\r" not in ln]
    lines = [ln for ln in lines if ln] + [""]  # an empty line, counted as the one before it
    src = write_sources(tmp_path / "src", files)
    stdin = ("\n".join(lines) + "\n").encode()
    steps = [("compile", compile_args(src, tmp_path / "system.dic.zst")),
             ("reorder", ["-i", tmp_path / "system.dic.zst", "-o", tmp_path / "reordered"]),
             ("map", ["-i", tmp_path / "system.dic.zst", "-m", tmp_path / "reordered", "-o", tmp_path / "mapped.dic.zst"])]
    for name, args in steps:
        p = run(name, *args, stdin=stdin)
        assert p.returncode == 0, (name, p.stderr.decode())
    new_l = {int(x.split("\t")[0]): k + 1 for k, x in enumerate((tmp_path / "reordered.lmap").read_text().splitlines())}
    new_r = {int(x.split("\t")[0]): k + 1 for k, x in enumerate((tmp_path / "reordered.rmap").read_text().splitlines())}
    out = {}
    for dic in ("system.dic.zst", "mapped.dic.zst"):
        for mode in ("mecab", "wakati", "detail"):
            p = run("tokenize", "-i", tmp_path / dic, "-O", mode, stdin=stdin)
            assert p.returncode == 0, p.stderr.decode()
            out[dic, mode] = p.stdout.decode()
    for mode in ("mecab", "wakati"):
        assert out["mapped.dic.zst", mode] == out["system.dic.zst", mode], mode
    before, after = out["system.dic.zst", "detail"].splitlines(), out["mapped.dic.zst", "detail"].splitlines()
    assert len(before) == len(after) and len(before) > len(lines)
    for a, b in zip(before, after):
        if a == "EOS":
            assert b == "EOS"
            continue
        (la, ra), (lb, rb) = detail_ids(a), detail_ids(b)
        assert (lb, rb) == (new_l[la], new_r[ra]), a
        strip = lambda s: [x for x in s.split("\t") if not x.startswith(("left_id=", "right_id="))]
        assert strip(a) == strip(b)
