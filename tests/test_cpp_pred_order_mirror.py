"""Builds and runs the known-answer tests of the C++ mirror's algo::OrderByPred (include/dgx_algo.hpp over dgx_pred_order)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp):
    exe = os.path.join(tmp, "test_pred_order_kat")
    subprocess.check_call([
        "g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
        os.path.join(ROOT, "tests", "cpp", "test_pred_order_kat.cpp"), "-o", exe,
        "-L", os.path.join(ROOT, "dgraph_b200"), "-ldgx", "-Wl,-rpath," + os.path.join(ROOT, "dgraph_b200"),
    ])
    return exe


def test_pred_order_mirror_compiles_and_links(tmp_path):
    _build(str(tmp_path))


@pytest.mark.gpu
def test_pred_order_mirror_known_answers(tmp_path):
    r = subprocess.run([_build(str(tmp_path))], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "OK: 0 failure(s)" in r.stdout, r.stdout + r.stderr
