"""`tokenize --boundary-marker C`: the marker parser (cli_common.hpp strip_boundary_markers), compiled on its own into
a small host program, so it runs without a device."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HARNESS = r"""
#include <iostream>
#include "cli_common.hpp"
int main(int argc, char** argv) {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::vector<uint32_t> b = cli::strip_boundary_markers(line, argv[1][0]);
        std::cout << line << '\t';
        for (size_t i = 0; i < b.size(); ++i) std::cout << (i ? "," : "") << b[i];
        std::cout << '\n';
    }
}
"""


@pytest.fixture(scope="module")
def parser(tmp_path_factory):
    cxx = shutil.which(os.environ.get("CXX", "c++")) or shutil.which("g++")
    if not cxx:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("marker")
    (d / "h.cpp").write_text(HARNESS)
    exe = d / "h"
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "vibrato_b200", "cpp"), "-I",
                           os.path.join(ROOT, "include"), str(d / "h.cpp"), "-o", str(exe)])

    def run(marker, lines):
        out = subprocess.run([str(exe), marker], input="\n".join(lines) + "\n", capture_output=True, text=True,
                             check=True).stdout
        res = []
        for row in out.splitlines():
            text, b = row.split("\t")
            res.append((text, [int(x) for x in b.split(",")] if b else []))
        return res

    return run


def test_marker_parser(parser):
    got = parser("|", ["京都|東京都|京都", "|a||b|", "abc", "", "||", "東京 | 都"])
    assert got == [
        ("京都東京都京都", [6, 15]),   # byte offsets in the line without markers
        ("ab", [0, 1, 2]),             # adjacent markers give one boundary; the ends give 0 and len
        ("abc", []),
        ("", []),
        ("", [0]),
        ("東京  都", [7]),
    ]


def test_other_marker_bytes(parser):
    assert parser("/", ["a/b|c"]) == [("ab|c", [1])]
    assert parser("*", ["**x*"]) == [("x", [0, 1])]
