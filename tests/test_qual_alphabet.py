"""The test helpers that choose BQSR kernel paths (tests/util.py): with_qual_alphabet and the restatements of the host's kernel choice."""
import numpy as np
import pytest

from elprep_b200 import synth
from util import SYNTH_QUALS, apply_plan, fast_plan, with_qual_alphabet


@pytest.mark.parametrize("values", [(30,), (2, 30), (5, 6), (3, 9, 41), (2, 11, 25, 37, 40), (0, 1, 2, 3, 4, 13, 22, 31), (2, 6, 15, 22, 27, 33, 37, 40)])
def test_with_qual_alphabet_is_monotone_and_exact(values):
    w = synth.make_workload(300, [("c", 50_000)], seed=7, want_reference=False)
    w2 = with_qual_alphabet(w, values, seed=3)
    q0, q1 = w.batch.qual, w2.batch.qual
    assert np.unique(q1).tolist() == sorted(values)
    for a, b in zip(SYNTH_QUALS[:-1], SYNTH_QUALS[1:]):          # every byte of a lower level maps at or below every byte of a higher one
        assert q1[q0 == a].max() <= q1[q0 == b].min()
    assert np.array_equal(with_qual_alphabet(w, values, seed=3).batch.qual, q1)
    assert np.array_equal(w.batch.qual, q0)                       # the input is not changed
    for f in ("flag", "pos", "lseq", "seq"):
        assert np.array_equal(getattr(w2.batch, f), getattr(w.batch, f))


def test_kernel_choice_restatements():
    assert fast_plan(SYNTH_QUALS, 4, 150) == (3, 0)
    assert fast_plan((2, 12, 23, 37, 45), 4, 151) == (4, 3)        # 45 and 37 share q & 7
    assert fast_plan((2, 12, 23, 37, 40), 4, 151) == (4, 0)
    assert fast_plan((5,), 4, 151) is None                          # no slot at all
    assert fast_plan((2, 11, 25, 37, 40), 32, 151) == (4, 0) and fast_plan((2, 11, 25, 37, 40), 33, 151) is None
    assert fast_plan(SYNTH_QUALS, 1, 1024) == (3, 0) and fast_plan(SYNTH_QUALS, 1, 1025) is None
    assert apply_plan(SYNTH_QUALS, 4, 151) == "v2" and apply_plan((2, 11, 25, 37, 40), 4, 151) == "gmem"
    assert apply_plan((2, 30), 1, 1024, 1024) == "v2" and apply_plan(SYNTH_QUALS, 4, 1024, 1024) == "gmem"
