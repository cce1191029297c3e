"""The branch-free division-by-constant, reciprocal and square-root sequences of the tri-lane kernels' scalar pre-pass
(cpi_b200/csrc/exact_math.cuh) equal the IEEE operations, bit for bit, on their stated domains: a C restatement with libm's fma()
against the host's correctly rounded division and sqrt, on random inputs in every binade (about 2e9 in all) and on hard cases
(significands 1 and all ones, results next to rounding midpoints), with perturbed hardware seeds."""
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
PER_BINADE = 300_000                    # x 3 primitives x ~2 000 binades


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    exe = str(tmp_path_factory.mktemp("exact_math") / "exact_math_check")
    base = [cc, "-O2", "-ffp-contract=off", os.path.join(HERE, "exact_math_check.c"), "-lm", "-o", exe]
    if subprocess.run(base[:3] + ["-fopenmp"] + base[3:], capture_output=True).returncode != 0:
        subprocess.run(base, check=True)            # no OpenMP: the same check on one thread
    return exe


def test_exact_primitives_match_ieee(checker):
    r = subprocess.run([checker, str(PER_BINADE)], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout + r.stderr
    assert ", 0 disagreements" in r.stdout
    assert int(r.stdout.split()[-4]) > 1_800_000_000, r.stdout
