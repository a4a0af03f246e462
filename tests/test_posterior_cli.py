"""`tokenize --posterior` and `evaluate --theta / --posterior` argument checks that need no device: each is a usage
error (status 2, before the dictionary is read)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "vibrato_b200", "bin")


def usage_error(exe, args, marker):
    path = os.path.join(BIN, exe)
    if not os.path.exists(path):
        pytest.skip("CLIs not built")
    p = subprocess.run([path] + args, input=b"x\n", capture_output=True, timeout=60)
    assert p.returncode == 2, p.stderr
    assert marker in p.stderr  # the usage text, not a failed dictionary load
    assert b"Loading" not in p.stderr


@pytest.mark.parametrize("args", [
    ["--posterior", "1"],                                    # needs -m -t
    ["--posterior", "1", "-t", "0.1"],                       # -t alone belongs to -m or --sample
    ["--posterior", "1", "-m"],                              # -m needs -t
    ["--posterior", "1", "-m", "-t", "0.1", "-a"],           # the posterior path or lattice nodes, not both
    ["--posterior", "1", "-m", "-t", "0.1", "--sample", "2"],
    ["--posterior", "1", "-m", "-t", "0.1", "--format-on", "host"],
    ["--posterior", "-1", "-m", "-t", "0.1"],
    ["--posterior", "inf", "-m", "-t", "0.1"],
    ["--posterior", "nan", "-m", "-t", "0.1"],
    ["--posterior", "1x", "-m", "-t", "0.1"],
    ["-m", "-t", "0.1", "--posterior"],                      # needs its value
])
def test_tokenize_usage_errors(tmp_path, args):
    usage_error("tokenize", ["-i", str(tmp_path / "missing")] + args, b"--posterior G")


@pytest.mark.parametrize("args", [
    ["--theta", "0.1"],                                      # each needs the other
    ["--posterior", "1"],
    ["--theta", "0", "--posterior", "1"],
    ["--theta", "-0.1", "--posterior", "1"],
    ["--theta", "0.1", "--posterior", "-1"],
    ["--theta", "0.1", "--posterior", "nan"],
    ["--theta", "x", "--posterior", "1"],
    ["--theta", "0.1", "--posterior"],
])
def test_evaluate_usage_errors(tmp_path, args):
    usage_error("evaluate", ["-i", str(tmp_path / "missing"), "-t", str(tmp_path / "corpus")] + args, b"--posterior G")
