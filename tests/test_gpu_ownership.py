"""Device and page-locked memory has one owner: every allocation a context makes is freed by elp_destroy, whatever the context did,
and elp_reset reruns reuse what the first run allocated.  elp_debug_live_allocations counts the allocations the library holds."""
import gc

import numpy as np
import pytest

import elsites_cases as ec
import fasta_cases as fc
from elprep_b200 import _lib, device, sam, synth
from samtext import sam_text
from test_gpu_bgzf_ingest import bam_file
from util import encode_bam, set_side_inputs

pytestmark = pytest.mark.gpu

SMALL = [("chr20", 600_000), ("chr21", 300_000), ("chrM", 16_569)]


def _live():
    gc.collect()   # contexts that other tests left to the collector are closed before the count is read
    return device.live_allocations()


def _write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


def _header(names):
    return sam.Header(sq=[{"SN": n, "LN": 1 << 30} for n in names])


@pytest.fixture(scope="module")
def inputs():
    """one workload, its reads cut in three: BAM records, SAM text and a BGZF-compressed BAM file"""
    w = synth.make_workload(1500, SMALL, seed=11)
    n = w.batch.n
    a, b = n // 3, 2 * n // 3
    raw, off = encode_bam(w.batch.take(np.arange(0, a)), w.header)
    text = sam_text(w.batch.take(np.arange(a, b)), w.header)
    raw3, _ = encode_bam(w.batch.take(np.arange(b, n)), w.header)
    return w, (raw, off), text, bam_file(w, raw3)


def _pipeline(ctx, w, bam, text, bgzf_data):
    """every ingest path, sort with optical duplicate marking, the target filter, BQSR and every fetch"""
    ctx.append_bam(*bam)
    ctx.append_sam(text)
    ctx.append_bgzf(bgzf_data)
    ctx.append_bgzf_end()
    ctx.set_output_filter(remove=["MD"])
    ctx.sort_markdup(device.SO_COORDINATE, _lib.MARKDUP_OPTICAL)
    ctx.filter_target_regions()
    ctx.bqsr_gather()
    ctx.bqsr_finalize()
    ctx.bqsr_apply()
    ctx.fetch()
    ctx.fetch_bam()
    ctx.fetch_sam()
    ctx.fetch_bgzf()


def _context(w):
    ctx = device.Context(w.header)
    set_side_inputs(ctx, w)
    ctx.set_target_regions(0, [[1, 200_000]])
    ctx.set_bqsr_target_regions(0, [[1, 300_000]])
    ctx.set_bqsr_target_regions(1, [[1, 300_000]])
    return ctx


def test_pipeline_frees_everything(inputs):
    w, bam, text, data = inputs
    base = _live()
    ctx = _context(w)
    try:
        _pipeline(ctx, w, bam, text, data)
        assert _live() > base
    finally:
        ctx.close()
    assert _live() == base


@pytest.mark.parametrize("chunk", [7, 0])
def test_loaders_accepted_and_refused(tmp_path, chunk):
    """accepted loads, then loads refused mid-file; every refusal leaves nothing behind once the context is destroyed"""
    base = _live()
    ctx = device.Context(_header(ec.NAMES))
    try:
        ctx.debug_set_sites_chunk(chunk)
        ctx.load_known_sites([_write(tmp_path, "good.elsites", ec.VALID[0][1][0])])
        for cid, files, _ in ec.INVALID:
            with pytest.raises(device.ElprepError):
                ctx.load_known_sites([_write(tmp_path, f"{cid}_{i}.elsites", f) for i, f in enumerate(files)])
    finally:
        ctx.close()
    assert _live() == base
    ctx = device.Context(_header(fc.NAMES))
    try:
        ctx.debug_set_reference_chunk(chunk)
        ctx.load_reference(_write(tmp_path, "good.fa", fc.FASTA_VALID[0][1]))
        for cid, data, _ in fc.FASTA_INVALID + fc.ELFASTA_INVALID:
            with pytest.raises(device.ElprepError):
                ctx.load_reference(_write(tmp_path, f"{cid}.bad", data))
    finally:
        ctx.close()
    assert _live() == base


def test_set_after_load_and_reloads(tmp_path):
    """elp_set_* replaces one contig of a loaded table; a reload replaces the whole table and the block of the load before"""
    base = _live()
    ctx = device.Context(_header(ec.NAMES))
    try:
        sites = [_write(tmp_path, f"s{i}.elsites", files[0]) for i, (_, files, _, _) in enumerate(ec.VALID[:3])]
        ctx.load_known_sites(sites[:1])
        ctx.set_known_sites(0, [[5, 9], [20, 30]])
        ctx.set_known_sites(1, [])
        after_set = _live()
        ctx.load_known_sites(sites[1:2])
        ctx.load_known_sites(sites[2:3])
        ctx.set_known_sites(0, [[5, 9]])
        assert _live() <= after_set   # the per-contig buffers of the first sets went with the reloads
        ref = _write(tmp_path, "r.fa", fc.FASTA_VALID[0][1])
        ctx.load_reference(ref)
        ctx.set_reference(0, np.frombuffer(b"ACGTN" * 40, np.uint8))
        ctx.load_reference(ref)
        ctx.set_reference(1, np.frombuffer(b"ACGT", np.uint8))
        ctx.load_reference(ref)
    finally:
        ctx.close()
    assert _live() == base


def test_reset_reruns_allocate_nothing_new(inputs, tmp_path):
    """three reset-and-rerun cycles of the pipeline and both loaders on one context: cycles 2 and 3 hold what cycle 1 held"""
    w, bam, text, data = inputs
    names = [s["SN"] for s in w.header.SQ]
    sites = _write(tmp_path, "w.elsites", b"# elsites format version 1.0\n" + b"".join(f"{n}\t{i * 100}\t{i * 100 + 5}\n".encode() for n in names for i in range(1, 50)))
    fasta = b""
    for ci, n in enumerate(names):
        bases = bytes(np.ascontiguousarray(w.contig_bases[ci], dtype=np.uint8))
        fasta += b">" + n.encode() + b"\n" + b"".join(bases[i:i + 60] + b"\n" for i in range(0, len(bases), 60))
    ref = _write(tmp_path, "w.fa", fasta)
    base = _live()
    ctx = _context(w)
    try:
        counts = []
        for _ in range(3):
            ctx.reset()
            ctx.load_known_sites([sites])
            ctx.load_reference(ref)
            _pipeline(ctx, w, bam, text, data)
            counts.append(_live())
        assert counts[1] == counts[0] and counts[2] == counts[0], counts
    finally:
        ctx.close()
    assert _live() == base
