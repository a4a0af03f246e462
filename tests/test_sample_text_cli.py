"""`tokenize --sample` argument checks that need no device: each is a usage error (status 2, before the dictionary
is read)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "vibrato_b200", "bin", "tokenize")


@pytest.mark.parametrize("args", [
    ["--sample", "3"],                                   # --sample needs -t
    ["-t", "0.1"],                                       # -t belongs to -m or --sample
    ["--sample", "3", "-t", "0.1", "--seed"],            # --seed needs its value
    ["--seed", "5", "-m", "-t", "0.1"],                  # --seed belongs to --sample
    ["--sample", "3", "-t", "0.1", "-a"],                # samples or lattice nodes, not both
    ["--sample", "3", "-t", "0.1", "--format-on", "host"],
    ["--sample", "0", "-t", "0.1"],
    ["--sample", "1025", "-t", "0.1"],
    ["--sample", "3x", "-t", "0.1"],
    ["--sample", "3", "-t", "0.1", "--seed", "-1"],
    ["--sample", "3", "-t", "0.1", "--seed", "18446744073709551616"],
])
def test_sample_usage_errors(tmp_path, args):
    if not os.path.exists(EXE):
        pytest.skip("CLIs not built")
    p = subprocess.run([EXE, "-i", str(tmp_path / "missing")] + args, input=b"x\n", capture_output=True, timeout=60)
    assert p.returncode == 2
    assert b"--sample N" in p.stderr  # the usage text, not a failed dictionary load
    assert b"Loading" not in p.stderr
