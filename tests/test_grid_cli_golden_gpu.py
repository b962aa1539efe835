"""Grid runs are unchanged by region features (DESIGN §26): evaluate's rank file and generate's results.json for a grid
checkpoint are byte for byte the files the build before region features wrote (tests/golden/grid_cli, made by
tests/golden/make_grid_cli_golden.py with that build)."""
import importlib.util
import os

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def test_grid_evaluate_and_generate_files_are_the_previous_builds(tmp_path):
    spec = importlib.util.spec_from_file_location("make_grid_cli_golden", os.path.join(GOLDEN, "make_grid_cli_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    mk.produce(str(tmp_path), ROOT)
    want = sorted(os.listdir(os.path.join(GOLDEN, "grid_cli")))
    assert sorted(os.listdir(str(tmp_path))) == want
    for name in want:
        with open(os.path.join(GOLDEN, "grid_cli", name), "rb") as a, open(str(tmp_path / name), "rb") as b:
            assert a.read() == b.read(), name
