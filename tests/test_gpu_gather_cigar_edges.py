"""GPU parity of the BQSR gather at its CIGAR edges (gather_cigar_cases.py): indels on every 16-base chunk and 32-base lane boundary, the
count kernel's record limits, shapes closed_form_clip rejects, 64 operations, the adaptor boundary swept across every operation, and reads
that end on or run past the last base of their contig.

Every family runs under a general QUAL alphabet (bqsr_prep -> bqsr_chunk / bqsr_chunk_list), a fast one (bqsr_prep2 -> bqsr_count /
bqsr_count_indel, the rest handed to bqsr_prep through cx_list), and the general one with --max-cycle below the longest reads (their bases
past max_cycle carry QUAL 2, and the gather takes them one warp per read).  Order, FLAG, table counters, EmpiricalQuality, report text and
QUAL bytes must equal the oracle's, and kernel_stats() must show the path each family is meant for.  Reads the oracle or the device refuse
run one per context, and the context must work again after elp_reset."""
import numpy as np
import pytest

import gather_cigar_cases as gc
from elprep_b200 import synth
from util import bqsr_paths, compare_bqsr, fast_plan, gpu_phases, gpu_pipeline, oracle_pipeline, oracle_tables_dense, set_side_inputs

pytestmark = pytest.mark.gpu

CONFIGS = ("general", "fast", "general_max_cycle")
MAX_CYCLE_BELOW = {"indel": 100, "indel_over_record": 100, "complex": 48, "adaptor": 48, "contig_end": 40}
_families = {}


def _family(name, config):
    if (name, config) not in _families:
        F = gc.family(name, gc.FAST if config == "fast" else gc.GENERAL, seed=7)
        mc = MAX_CYCLE_BELOW[name] if config == "general_max_cycle" else 500
        if mc < 500:
            F = gc.Family(gc.cap_cycles(F.good, mc), F.names, [(n, gc.cap_cycles(w, mc), o, d) for n, w, o, d in F.errors])
            assert int(F.good.batch.lseq.max()) > mc
        _families[(name, config)] = (F, mc)
    return _families[(name, config)]


def _check_paths(name, config, st):
    assert bqsr_paths(st)[0] == ("fast" if config == "fast" else "general"), sorted(st)
    ran = set(st)
    indel_records = "bqsr_g_count_indel" in st and st["bqsr_g_count_indel"]["alg_bytes"] > 0   # (bytes of the indel records it read)
    if config == "general_max_cycle":
        assert "bqsr_g_warp_per_read" in ran, sorted(st)
        return
    assert "bqsr_g_warp_per_read" not in ran, sorted(st)
    if config == "general":
        assert "bqsr_g_chunk_list" in ran, sorted(st)                 # every family has reads with an indel or a trailing deletion
    else:
        assert ("bqsr_g_chunk_list" in ran) == (name != "indel"), sorted(st)   # the reads handed to the general kernels
        if name == "indel":                                            # every read is one indel record of the count kernel
            assert indel_records and "bqsr_g_prep" not in ran, sorted(st)
        elif name in ("indel_over_record", "complex"):                 # every read is handed to the general kernels
            assert not indel_records and "bqsr_g_prep" in ran, sorted(st)
        elif name == "adaptor":                                        # both: the boundary outside / inside an indel read's alignment
            assert indel_records and "bqsr_g_prep" in ran, sorted(st)
        else:
            assert "bqsr_g_prep" in ran, sorted(st)


def _column(c, mc):
    if c == 0:
        return "QualityScore"
    if c <= 2 * mc + 1:
        return f"Cycle {c - 1 - mc}"
    return f"Context {c - 2 * mc - 2}"


def _tables_message(F, g, d, mc):
    """the differing cells (read group covariate, QUAL, column) and the family's reads that contribute to them, from the oracle run once
    per candidate read"""
    b = F.good.batch
    cells = sorted({(int(cv), int(q), int(c)) for cv, q, c, _ in np.argwhere(g["tables"] != d)})
    rg_cov, cov_names = F.good.header.rg_cov_ids()
    qo = b.qual_off.astype(np.int64)
    covs, quals = {c[0] for c in cells[:20]}, {c[1] for c in cells[:20]}
    cand = [i for i in range(b.n) if b.rg[i] >= 0 and rg_cov[b.rg[i]] in covs and quals & set(np.unique(b.qual[qo[i]:qo[i + 1]]).tolist())]
    contrib = gc.contributions(F.good, mc, cand[:400])
    lines = [f"{len(cells)} table cells differ"]
    for cv, q, c in cells[:20]:
        who = [F.names[i] for i, t in contrib.items() if t[cv, q, c].any()]
        lines.append(f"  {cov_names[cv]} QUAL {q} {_column(c, mc)}: device {g['tables'][cv, q, c].tolist()} oracle {d[cv, q, c].tolist()}; "
                     f"reads: {', '.join(who[:12])}{' ...' if len(who) > 12 else ''}")
    return "\n".join(lines)


@pytest.mark.parametrize("config", CONFIGS)
@pytest.mark.parametrize("name", gc.FAMILIES)
def test_family_parity(name, config):
    F, mc = _family(name, config)
    g = gpu_pipeline(F.good, max_cycle=mc, profile=True)
    o = oracle_pipeline(F.good, max_cycle=mc)
    d, _ = oracle_tables_dense(o["tables"], mc)
    if not np.array_equal(g["tables"], d):
        pytest.fail(_tables_message(F, g, d, mc))
    compare_bqsr(g, o, mc)
    _check_paths(name, config, g["stats"])


@pytest.mark.parametrize("config", CONFIGS)
@pytest.mark.parametrize("name", ["complex", "adaptor", "contig_end"])
def test_error_reads(name, config):
    """each refused read alone in a context: the device's error code (ELP_ELIMIT for 65 operations, which the oracle accepts; ELP_ECLIP
    and ELP_EREFEND where the oracle fails too), no tables, and after elp_reset the same context gathers a few good reads of the family"""
    from elprep_b200 import device
    F, mc = _family(name, config)
    assert F.errors
    probe = synth.Workload(F.good.header, F.good.batch.take(np.arange(min(30, F.good.batch.n))), F.good.contig_bases, F.good.sites, {})
    o_probe = oracle_pipeline(probe, max_cycle=mc)
    n_cov = len(F.good.header.rg_cov_ids()[1])
    for n, w, ocode, dcode in F.errors:
        ctx = device.Context(w.header, max_cycle=mc, profile=True)
        try:
            set_side_inputs(ctx, w)
            ctx.append(w.batch)
            ctx.sort_markdup()
            with pytest.raises(device.ElprepError) as ei:
                ctx.bqsr_gather()
            assert ei.value.code == dcode, (n, ei.value.code, str(ei.value))
            st = ctx.kernel_stats()
            assert "bqsr_g_prep" in st, (n, sorted(st))                # both gathers reach bqsr_prep_kernel with these reads
            fast = fast_plan(np.unique(w.batch.qual).tolist(), n_cov, int(w.batch.lseq.max())) is not None
            assert ("bqsr_g_count" in st) == fast, (n, sorted(st))
            with pytest.raises(device.ElprepError) as ei:
                ctx.bqsr_finalize(None)
            assert ei.value.code == -16, n
            ctx.reset()
            ctx.reset_stats()
            ctx.append(probe.batch)
            g = gpu_phases(ctx, profile=True)
        finally:
            ctx.close()
        compare_bqsr(g, o_probe, mc)
