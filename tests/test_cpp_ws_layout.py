"""Builds and runs the known-answer tests of dgraph_b200/csrc/ws_layout.hpp, the layout every per-call device workspace
of libdgx is carved by: section order, alignment, offsets against the total, and each section's extent."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ws_layout_known_answers(tmp_path):
    exe = os.path.join(str(tmp_path), "test_ws_layout")
    subprocess.check_call([
        "g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "dgraph_b200", "csrc"),
        os.path.join(ROOT, "tests", "cpp", "test_ws_layout.cpp"), "-o", exe,
    ])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and "OK: 0 failure(s)" in r.stdout, r.stdout + r.stderr
