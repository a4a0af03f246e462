"""`tokenize -a/--all-morphs` argument checks that need no device: -a renders nodes on the device only, so with
--format-on host it is a usage error (status 2, before the dictionary is read)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "vibrato_b200", "bin", "tokenize")


@pytest.mark.parametrize("flag", ["-a", "--all-morphs"])
def test_all_morphs_format_on_host_is_a_usage_error(tmp_path, flag):
    if not os.path.exists(EXE):
        pytest.skip("CLIs not built")
    p = subprocess.run([EXE, "-i", str(tmp_path / "missing"), flag, "--format-on", "host"], input=b"x\n",
                       capture_output=True, timeout=60)
    assert p.returncode == 2
    assert b"--all-morphs" in p.stderr  # the usage text
