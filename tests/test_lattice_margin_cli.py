"""`tokenize --cost-margin` argument checks that need no device: each is a usage error (status 2, before the
dictionary is read)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "vibrato_b200", "bin", "tokenize")


@pytest.mark.parametrize("args", [
    ["--cost-margin", "5"],                              # needs -a
    ["--cost-margin", "0", "-O", "wakati"],
    ["-a", "--cost-margin", "-1"],                       # negative
    ["-a", "--cost-margin", "1x"],                       # not a number
    ["-a", "--cost-margin", ""],
    ["-a", "--cost-margin", str((1 << 62) + 1)],        # above 2^62
    ["-a", "--cost-margin", "18446744073709551616"],
    ["-a", "--cost-margin"],                             # no value
])
def test_cost_margin_usage_errors(tmp_path, args):
    if not os.path.exists(EXE):
        pytest.skip("CLIs not built")
    p = subprocess.run([EXE, "-i", str(tmp_path / "missing")] + args, input=b"x\n", capture_output=True, timeout=60)
    assert p.returncode == 2
    assert b"--cost-margin D" in p.stderr  # the usage text, not a failed dictionary load
    assert b"Loading" not in p.stderr


def test_cost_margin_accepted_with_all_morphs(tmp_path):
    """-a --cost-margin 2^62 passes the usage checks: the run gets as far as loading the (missing) dictionary."""
    if not os.path.exists(EXE):
        pytest.skip("CLIs not built")
    p = subprocess.run([EXE, "-i", str(tmp_path / "missing"), "-a", "--cost-margin", str(1 << 62)], input=b"x\n",
                       capture_output=True, timeout=60)
    assert p.returncode != 2 and b"Loading" in p.stderr
