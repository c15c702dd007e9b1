"""The numpy mirrors of the batch-wide statistics (cluster-log and job-log ensembles, power profile, paired comparison)
recomputed on the seeded inputs of tests/golden/make_golden_stats.py and compared byte for byte with the CSVs it wrote:
a change in the last bit of a mean, std, min, max or quantile fails here."""
import importlib.util
import os

import pytest

from conftest import GOLDEN_DIR

_spec = importlib.util.spec_from_file_location("make_golden_stats", os.path.join(GOLDEN_DIR, "make_golden_stats.py"))
GS = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(GS)


def test_every_fixture_has_a_case():
    assert sorted(os.listdir(GS.OUT_DIR)) == sorted(GS.CASES)


@pytest.mark.parametrize("name", sorted(GS.CASES))
def test_statistics_are_bit_identical_to_the_fixture(name, tmp_path):
    path = tmp_path / name
    GS.CASES[name](str(path))
    with open(os.path.join(GS.OUT_DIR, name), "rb") as f:
        want = f.read()
    assert path.read_bytes() == want
