"""BQSR finalize on the device (bqsr_finalize.cu: fin_emp, fin_tail, fin_lut, fin_clut) against the oracle, on synthetic tables.

The tables go in through tables_put, so every corner of the arithmetic can be reached without a workload that produces it: counts past
the maxObs clamp (the Round path of Entry), mis = 0 and mis = obs, priors more than 20 away from the estimate, estimates that clamp at
93, QUAL values without any table entry, a read group whose table is empty, quantize levels 0 / 1 / 16 / 94, static quantization with one
and with several values, --max-cycle 1 and 500, and enough covariates that the compact apply table exceeds 80 KB.  EmpiricalQuality,
the recalibration report text (when one is asked for) and every recalibrated QUAL byte must equal the oracle's."""
import os
import tempfile

import numpy as np
import pytest

from elprep_b200 import synth
from util import apply_plan, bqsr_paths, with_qual_alphabet

pytestmark = pytest.mark.gpu

CONTIGS = [("chr20", 300_000), ("chr21", 100_000)]
MAX_OBS = 2147483647 - 1


def synthetic_tables(n_cov, max_cycle, quals, rng, empty_cov=None, huge=True):
    """dense [n_cov][94][1 + (2 max_cycle + 1) + 16][2] tables with rows for the QUAL values ``quals`` only"""
    ncol = 1 + (2 * max_cycle + 1) + 16
    t = np.zeros((n_cov, 94, ncol, 2), np.int64)
    for cv in range(n_cov):
        if cv == empty_cov:
            continue
        for q in quals:
            fill = rng.random(ncol) < 0.6
            obs = rng.integers(1, 5000, ncol)
            mis = (obs * rng.choice([0.0, 0.001, 0.01, 0.2, 0.5, 1.0], ncol)).astype(np.int64)   # 0 and obs included
            obs[0] = rng.integers(1, 10**7)
            mis[0] = int(obs[0] * rng.choice([0.0, 0.0005, 0.02, 0.3]))
            if huge and rng.random() < 0.5:      # past maxObs: k is rescaled with Round
                k = rng.integers(1, ncol, 4)
                obs[k] = rng.integers(MAX_OBS, 4 * MAX_OBS, 4)
                mis[k] = (obs[k] * rng.choice([0.0, 1e-4, 0.5], 4)).astype(np.int64)
                obs[0] = 5 * MAX_OBS
            fill[0] = True
            t[cv, q, :, 0] = np.where(fill, obs, 0)
            t[cv, q, :, 1] = np.where(fill, mis, 0)
    return t


def oracle_tables(dense, max_cycle):
    import oracle
    n_cov = dense.shape[0]
    nc = 2 * max_cycle + 1
    t = oracle.OracleTables(n_cov, max_cycle)
    t.q_obs[:, :94] = dense[:, :, 0, 0]; t.q_mis[:, :94] = dense[:, :, 0, 1]
    t.c_obs[:, :94] = dense[:, :, 1:1 + nc, 0]; t.c_mis[:, :94] = dense[:, :, 1:1 + nc, 1]
    t.x_obs[:, :94] = dense[:, :, 1 + nc:, 0]; t.x_mis[:, :94] = dense[:, :, 1 + nc:, 1]
    oracle.bqsr_finalize(t)
    emp = np.zeros(dense.shape[:3], np.uint8)
    emp[:, :, 0] = t.q_emp[:, :94]; emp[:, :, 1:1 + nc] = t.c_emp[:, :94]; emp[:, :, 1 + nc:] = t.x_emp[:, :94]
    return t, emp


def run(w, dense, max_cycle=500, quantize_levels=0, sqq=None, report=True, apply=True):
    """tables_put -> finalize -> (append -> sort -> apply) on the device and through the oracle; both results"""
    import oracle
    from elprep_b200 import device
    t, o_emp = oracle_tables(dense, max_cycle)
    o = {"emp": o_emp}
    ctx = device.Context(w.header, max_cycle=max_cycle, quantize_levels=quantize_levels, sqq=sqq, profile=True)
    g = {}
    try:
        ctx.tables_put(dense)
        with tempfile.TemporaryDirectory() as d:
            if report:
                p = os.path.join(d, "g.recal")
                ctx.bqsr_finalize(p)
                g["report"] = open(p).read()
                q = os.path.join(d, "o.recal")
                oracle.bqsr_report(t, oracle.OracleHeader(w.header).cov_names, q)
                o["report"] = open(q).read()
            else:
                ctx.bqsr_finalize(None)
        g["emp"] = ctx.empirical_get()
        if apply:
            ctx.append(w.batch)
            ctx.sort_markdup()
            ctx.bqsr_apply()
            idx, flag, qoff, qual = ctx.fetch()
            g["qual"] = qual[:int(qoff[-1])]
            g["apply"] = bqsr_paths(ctx.kernel_stats())[1]
            assert g["apply"] == apply_plan(w.params["quals"], dense.shape[0], int(w.batch.lseq.max()), max_cycle)
            b = w.batch.copy()
            oracle.mark_duplicates(b, w.header, n_threads=1)
            srt = b.take(oracle.coordinate_sort(b, n_threads=4))
            oracle.bqsr_apply(srt, w.header, t, quantize_levels=quantize_levels, sqq=sqq, n_threads=4)
            o["qual"] = srt.qual
            assert np.array_equal(qoff, srt.qual_off)
    finally:
        ctx.close()
    return g, o


def check(g, o):
    assert np.array_equal(g["emp"], o["emp"]), "EmpiricalQuality differs"
    if "report" in g:
        assert g["report"] == o["report"], "recalibration report text differs"
    if "qual" in g:
        assert np.array_equal(g["qual"], o["qual"]), "QUAL bytes differ"


VALUES = (2, 12, 23, 37, 45)      # four slots: the compact table of 4 covariates exceeds 80 KB (global-table kernel)
SMALL = (2, 12, 23, 45)           # three slots: bqsr_apply2_kernel over the compact table


def workload(seed, n_rg=4, values=VALUES, L=151):
    return with_qual_alphabet(synth.make_workload(1_500, CONTIGS, seed=seed, L=L, n_rg=n_rg), values)


@pytest.mark.parametrize("levels", [0, 1, 16, 94])
def test_quantize_levels(levels):
    """45 occurs in the reads but has no table row (never observed); read group 2 has an empty table"""
    w = workload(9100 + levels)
    rng = np.random.default_rng(levels)
    dense = synthetic_tables(4, 500, (2, 12, 23, 37, 60, 93), rng, empty_cov=2)
    g, o = run(w, dense, quantize_levels=levels)
    check(g, o)


@pytest.mark.parametrize("sqq", [[20], [10, 20, 30], [7, 40, 93]])
def test_static_quantization(sqq):
    w = workload(9200 + len(sqq), values=SMALL)
    dense = synthetic_tables(4, 500, (12, 23, 37), np.random.default_rng(sum(sqq)))
    for levels in (0, 16):
        g, o = run(w, dense, quantize_levels=levels, sqq=np.array(sqq, np.uint8), report=levels == 0)
        check(g, o)


def test_extreme_counts():
    """every cell of a row at the maxObs clamp, mis = 0 / mis = obs across the QUAL range, priors far from the estimate (QUAL 60 with
    half the bases wrong), estimates that clamp at 93 (QUAL 93 with no errors at all); the reads' QUAL 45 has no row"""
    w = workload(9300, values=SMALL)
    ncol = 1 + 1001 + 16
    dense = np.zeros((4, 94, ncol, 2), np.int64)
    dense[0, 12, :, 0] = np.arange(ncol) * 997 + 3 * MAX_OBS; dense[0, 12, :, 1] = dense[0, 12, :, 0] // 3
    dense[0, 23, :, 0] = 1000; dense[0, 23, :, 1] = 0
    dense[0, 37, :, 0] = 1000; dense[0, 37, :, 1] = 1000
    dense[1, 60, :, 0] = 2000; dense[1, 60, :, 1] = 1000
    dense[1, 93, :, 0] = 10**9; dense[1, 93, :, 1] = 0
    dense[1, 12, :, 0] = 10**6; dense[1, 12, :, 1] = 0
    dense[2, 37, 0, 0] = 10; dense[2, 37, 0, 1] = 10            # only the QUAL row
    dense[3, 23, :, 0] = np.arange(ncol) % 7; dense[3, 23, :, 1] = (np.arange(ncol) % 7) // 2
    for levels in (0, 16):
        g, o = run(w, dense, quantize_levels=levels)
        check(g, o)


@pytest.mark.parametrize("max_cycle", [1, 500])
def test_max_cycle(max_cycle):
    """max_cycle 1: EmpiricalQuality and the report only (every 151-base read exceeds it)"""
    w = workload(9400 + max_cycle, values=SMALL)
    dense = synthetic_tables(4, max_cycle, (12, 23, 37), np.random.default_rng(max_cycle))
    g, o = run(w, dense, max_cycle=max_cycle, apply=max_cycle >= 151)
    check(g, o)


@pytest.mark.parametrize("n_rg", [9, 24])
def test_many_covariates(n_rg):
    """the compact apply table of 9 covariates x 4 slots x 151 cycles exceeds 80 KB: the global-table kernel runs"""
    w = workload(9500 + n_rg, n_rg=n_rg)
    dense = synthetic_tables(n_rg, 500, (2, 12, 23, 37), np.random.default_rng(n_rg), empty_cov=n_rg - 1, huge=False)
    g, o = run(w, dense)
    check(g, o)
    assert g["apply"] == apply_plan(VALUES, n_rg, 151) == "gmem"


def test_without_report_and_reuse():
    """finalize without a report keeps everything on the device; a second tables_put -> finalize on the same context recomputes it"""
    from elprep_b200 import device
    w = workload(9600)
    d1 = synthetic_tables(4, 500, (12, 23, 37), np.random.default_rng(1))
    d2 = synthetic_tables(4, 500, (2, 23, 45), np.random.default_rng(2), empty_cov=0)
    ctx = device.Context(w.header)
    try:
        for d in (d1, d2):
            ctx.tables_put(d)
            ctx.bqsr_finalize(None)
            assert np.array_equal(ctx.empirical_get(), oracle_tables(d, 500)[1])
    finally:
        ctx.close()
    g, o = run(w, d2, report=False)
    check(g, o)
