// Package gpu binds libelprep_b200.so (include/elprep_b200.h) under elPrep's own pipeline types: DeviceSam implements
// sam.PipelineOutput and sam.PipelineInput next to *sam.Sam (sam/filter-pipeline.go:33-61, 108-128, 242-279), and the
// operators of the path keep the reference's names and signatures (filters/mark-duplicates.go:406, filters/bqsr.go:467,677,936,
// filters/print-bqsr.go:269,300-329, filters/mark-optical-duplicates.go:468,601,701-731).
//
// STATUS: complete source, NOT COMPILED -- the image this repository is built in has no Go toolchain.  The same C entry points are
// exercised through ctypes (elprep_b200/device.py, tests/) and from plain C (tests/c/cabi_client.c).
//
// Build inside the elPrep tree:  CGO_CFLAGS=-I<repo>/include CGO_LDFLAGS="-L<repo>/elprep_b200/lib -lelprep_b200" go build ./...
package gpu

/*
#cgo LDFLAGS: -lelprep_b200
#include <stdlib.h>
#include "elprep_b200.h"
*/
import "C"

import (
	"log"
	"runtime"
	"sync"
	"unsafe"

	"github.com/exascience/elprep/v5/filters"
	"github.com/exascience/elprep/v5/sam"
	"github.com/exascience/elprep/v5/utils"
	"github.com/exascience/elprep/v5/utils/nibbles"
	"github.com/exascience/pargo/pipeline"
)

// Options are the `elprep filter` flags the device path needs at creation (cmd/filter.go:435-481).
type Options struct {
	Device                       int
	MaxCycle, QuantizeLevels     int
	SQQ                          []uint8
	TablenamePrefix              string
	OpticalDuplicatesPixelDist   int
	MarkDuplicates, AlsoOpticals bool
}

// DeviceSam holds one elp_ctx: the reads of one (*sam.Sam) on one GPU.
type DeviceSam struct {
	ctx    *C.elp_ctx
	Header *sam.Header
	opts   Options
	mu     sync.Mutex
	alns   []*sam.Alignment // arrival order; the device returns indices into it
	refid  map[string]int32 // RNAME -> index in @SQ (filters.AddREFID, filters/simple-filters.go:208-231)
	rgIdx  map[string]int32 // RG:Z value -> index in @RG
}

func check(ctx *C.elp_ctx, rc C.int) {
	if rc != 0 {
		log.Panic(C.GoString(C.elp_last_error(ctx))) // the texts the reference panics with
	}
}

func cstrings(vals []string, null []bool) (**C.char, func()) {
	arr := C.malloc(C.size_t(len(vals)+1) * C.size_t(unsafe.Sizeof(uintptr(0))))
	ptrs := (*[1 << 28]*C.char)(arr)[: len(vals)+1 : len(vals)+1]
	for i, v := range vals {
		if null != nil && null[i] {
			ptrs[i] = nil
		} else {
			ptrs[i] = C.CString(v)
		}
	}
	return (**C.char)(arr), func() {
		for i := range vals {
			if ptrs[i] != nil {
				C.free(unsafe.Pointer(ptrs[i]))
			}
		}
		C.free(arr)
	}
}

// NewDeviceSam creates the context from the header tables the filters read: @SQ SN/LN, @RG ID/LB/PU.
func NewDeviceSam(header *sam.Header, opts Options) *DeviceSam {
	d := &DeviceSam{Header: header, opts: opts, refid: make(map[string]int32), rgIdx: make(map[string]int32)}
	names := make([]string, len(header.SQ))
	lens := make([]C.int32_t, len(header.SQ)+1)
	for i, sq := range header.SQ {
		names[i] = sq["SN"]
		lens[i] = C.int32_t(sam.SQLN(sq))
		d.refid[sq["SN"]] = int32(i)
	}
	ids, lbs, pus := make([]string, len(header.RG)), make([]string, len(header.RG)), make([]string, len(header.RG))
	noLB, noPU := make([]bool, len(header.RG)), make([]bool, len(header.RG))
	for i, rg := range header.RG {
		ids[i] = rg["ID"]
		d.rgIdx[rg["ID"]] = int32(i)
		lbs[i], noLB[i] = rg["LB"], rg["LB"] == ""
		_, hasPU := rg["PU"]
		_, hasID := rg["ID"]
		pus[i], noPU[i] = rg["PU"], !hasPU || !hasID // an @RG without ID: ID "" and no PU, so that the BQSR covariate is "" (readGroupCovariate, filters/bqsr.go:35-51)
	}
	cNames, f1 := cstrings(names, nil)
	cIDs, f2 := cstrings(ids, nil)
	cLBs, f3 := cstrings(lbs, noLB)
	cPUs, f4 := cstrings(pus, noPU)
	defer f1()
	defer f2()
	defer f3()
	defer f4()
	prefix := C.CString(opts.TablenamePrefix)
	defer C.free(unsafe.Pointer(prefix))
	var cfg C.elp_config
	cfg.device = C.int32_t(opts.Device)
	cfg.n_contigs = C.int32_t(len(header.SQ))
	cfg.contig_names = cNames
	cfg.contig_lengths = &lens[0]
	cfg.n_read_groups = C.int32_t(len(header.RG))
	cfg.rg_id, cfg.rg_lb, cfg.rg_pu = cIDs, cLBs, cPUs
	cfg.max_cycle = C.int32_t(opts.MaxCycle)
	cfg.quantize_levels = C.int32_t(opts.QuantizeLevels)
	if len(opts.SQQ) > 0 {
		cfg.sqq = (*C.uint8_t)(unsafe.Pointer(&opts.SQQ[0]))
		cfg.n_sqq = C.int32_t(len(opts.SQQ))
	}
	cfg.tablename_prefix = prefix
	cfg.optical_pixel_distance = C.int32_t(opts.OpticalDuplicatesPixelDist)
	if rc := C.elp_create(&cfg, &d.ctx); rc != 0 {
		log.Panic(C.GoString(C.elp_last_error(nil)))
	}
	runtime.SetFinalizer(d, func(d *DeviceSam) { C.elp_destroy(d.ctx) })
	return d
}

// columns of one batch, in the layout of elp_batch
type columns struct {
	refid, pos, nref, pnext, tlen, rg, lseq []int32
	flag                                    []uint16
	mapq, qname, seq, qual, opt             []byte
	qnameOff, cigarOff                      []uint64
	cigar                                   []uint32
}

var srTag = utils.Intern("sr")
var cigarCode = map[byte]uint32{'M': 0, 'I': 1, 'D': 2, 'N': 3, 'S': 4, 'H': 5, 'P': 6, '=': 7, 'X': 8}

func (d *DeviceSam) lookupRef(name string) int32 {
	if id, ok := d.refid[name]; ok {
		return id
	}
	return -1 // "*" or a name that is not an @SQ
}

// marshal turns []*sam.Alignment into columns (what a pargo stage does per batch, sam/filter-pipeline.go:92-104).
func (d *DeviceSam) marshal(batch []*sam.Alignment) *columns {
	n := len(batch)
	c := &columns{refid: make([]int32, n), pos: make([]int32, n), nref: make([]int32, n), pnext: make([]int32, n), tlen: make([]int32, n), rg: make([]int32, n),
		lseq: make([]int32, n), flag: make([]uint16, n), mapq: make([]byte, n), opt: make([]byte, n), qnameOff: make([]uint64, n+1), cigarOff: make([]uint64, n+1)}
	for i, aln := range batch {
		c.refid[i] = d.lookupRef(aln.RNAME)
		if aln.RNEXT == "=" {
			c.nref[i] = c.refid[i]
		} else {
			c.nref[i] = d.lookupRef(aln.RNEXT)
		}
		c.pos[i], c.pnext[i], c.tlen[i], c.flag[i], c.mapq[i] = aln.POS, aln.PNEXT, aln.TLEN, aln.FLAG, aln.MAPQ
		c.rg[i] = -1
		if rg := aln.RG(); rg != nil {
			if k, ok := d.rgIdx[rg.(string)]; ok {
				c.rg[i] = k
			}
		}
		if _, found := aln.TAGS.Get(srTag); found {
			c.opt[i] = C.ELP_OPT_SR
		}
		c.qname = append(c.qname, aln.QNAME...)
		c.qnameOff[i+1] = uint64(len(c.qname))
		for _, op := range aln.CIGAR {
			c.cigar = append(c.cigar, uint32(op.Length)<<4|cigarCode[op.Operation])
		}
		c.cigarOff[i+1] = uint64(len(c.cigar))
		l, off, raw := nibbles.Nibbles(aln.SEQ).ReflectValue()
		c.lseq[i] = int32(l)
		if off == 0 {
			c.seq = append(c.seq, raw[:(l+1)/2]...) // already BAM nibbles, first base in the high nibble
		} else {
			for k := 0; k < l; k += 2 { // a sliced sequence: re-pack from its first nibble
				b := aln.SEQ.Slice(k, k+1)
				hi := nibbles.Nibbles(b).Get(0) << 4
				if k+1 < l {
					hi |= nibbles.Nibbles(aln.SEQ).Get(k + 1)
				}
				c.seq = append(c.seq, hi)
			}
		}
		c.qual = append(c.qual, aln.QUAL...)
	}
	if len(c.cigar) == 0 {
		c.cigar = make([]uint32, 1)
	}
	if len(c.qname) == 0 {
		c.qname = make([]byte, 1)
	}
	if len(c.seq) == 0 {
		c.seq, c.qual = make([]byte, 1), make([]byte, 1)
	}
	return c
}

func (d *DeviceSam) appendBatch(batch []*sam.Alignment) {
	if len(batch) == 0 {
		return
	}
	c := d.marshal(batch)
	var b C.elp_batch
	b.n = C.uint64_t(len(batch))
	b.refid = (*C.int32_t)(unsafe.Pointer(&c.refid[0]))
	b.pos = (*C.int32_t)(unsafe.Pointer(&c.pos[0]))
	b.flag = (*C.uint16_t)(unsafe.Pointer(&c.flag[0]))
	b.mapq = (*C.uint8_t)(unsafe.Pointer(&c.mapq[0]))
	b.nref = (*C.int32_t)(unsafe.Pointer(&c.nref[0]))
	b.pnext = (*C.int32_t)(unsafe.Pointer(&c.pnext[0]))
	b.tlen = (*C.int32_t)(unsafe.Pointer(&c.tlen[0]))
	b.rg = (*C.int32_t)(unsafe.Pointer(&c.rg[0]))
	b.qname_off = (*C.uint64_t)(unsafe.Pointer(&c.qnameOff[0]))
	b.qname = (*C.uint8_t)(unsafe.Pointer(&c.qname[0]))
	b.cigar_off = (*C.uint64_t)(unsafe.Pointer(&c.cigarOff[0]))
	b.cigar = (*C.uint32_t)(unsafe.Pointer(&c.cigar[0]))
	b.l_seq = (*C.int32_t)(unsafe.Pointer(&c.lseq[0]))
	b.seq = (*C.uint8_t)(unsafe.Pointer(&c.seq[0]))
	b.qual = (*C.uint8_t)(unsafe.Pointer(&c.qual[0]))
	b.opt_flags = (*C.uint8_t)(unsafe.Pointer(&c.opt[0]))
	// elp_batch holds Go pointers to Go memory: pass it by value through a pinned call (cgo pointer rules: the library copies before returning)
	var pin runtime.Pinner
	for _, p := range []unsafe.Pointer{unsafe.Pointer(b.refid), unsafe.Pointer(b.pos), unsafe.Pointer(b.flag), unsafe.Pointer(b.mapq), unsafe.Pointer(b.nref), unsafe.Pointer(b.pnext),
		unsafe.Pointer(b.tlen), unsafe.Pointer(b.rg), unsafe.Pointer(b.qname_off), unsafe.Pointer(b.qname), unsafe.Pointer(b.cigar_off), unsafe.Pointer(b.cigar), unsafe.Pointer(b.l_seq),
		unsafe.Pointer(b.seq), unsafe.Pointer(b.qual), unsafe.Pointer(b.opt_flags)} {
		pin.Pin(p)
	}
	defer pin.Unpin()
	d.mu.Lock() // the arrival index the device hands back is the position in d.alns
	d.alns = append(d.alns, batch...)
	rc := C.elp_append_batch(d.ctx, &b)
	d.mu.Unlock()
	check(d.ctx, rc)
}

// AppendBgzf hands over the next bytes of a BGZF-compressed BAM file as they come off disk, cut anywhere; the device inflates them,
// walks the header and frames and ingests the records (elp_append_bgzf).  AppendBgzfEnd ends the file (EOF marker, no bytes left).
func (d *DeviceSam) AppendBgzf(chunk []byte) {
	if len(chunk) == 0 {
		return
	}
	d.mu.Lock()
	rc := C.elp_append_bgzf(d.ctx, (*C.uint8_t)(unsafe.Pointer(&chunk[0])), C.uint64_t(len(chunk)))
	d.mu.Unlock()
	check(d.ctx, rc)
}

func (d *DeviceSam) AppendBgzfEnd() {
	d.mu.Lock()
	rc := C.elp_append_bgzf_end(d.ctx)
	d.mu.Unlock()
	check(d.ctx, rc)
}

// FetchBgzf: output records [first, first+n) of elp_fetch_bam behind prefix (the BAM header on a file's first call) as BGZF blocks,
// deflated on the device (elp_fetch_bgzf), with the EOF marker when eof.  The bytes go to the file as they are, with no bgzf.Writer;
// the outputs of consecutive ranges, eof on the last only, make one file.
func (d *DeviceSam) FetchBgzf(first, n uint64, prefix []byte, eof bool) []byte {
	var records uint64
	if n > 0 {
		records = uint64(C.elp_fetch_bam_bytes(d.ctx, C.uint64_t(first), C.uint64_t(n))) // (0 on a refusal, which elp_fetch_bgzf then reports)
	}
	out := make([]byte, uint64(C.elp_bgzf_deflate_bound(C.uint64_t(records+uint64(len(prefix))))))
	var pp *C.uint8_t
	if len(prefix) > 0 {
		pp = (*C.uint8_t)(unsafe.Pointer(&prefix[0]))
	}
	e := C.int(0)
	if eof {
		e = 1
	}
	var got C.uint64_t
	check(d.ctx, C.elp_fetch_bgzf(d.ctx, C.uint64_t(first), C.uint64_t(n), pp, C.uint64_t(len(prefix)), e, (*C.uint8_t)(unsafe.Pointer(&out[0])),
		C.uint64_t(len(out)), &got))
	return out[:uint64(got)]
}

// AddNodes: the receiving end of phase 1 (sam/filter-pipeline.go:108-128).  The Finalize runs what By(CoordinateLess).ParallelStableSort
// (sam/sam-types.go:599-641) and filters.MarkDuplicates (+ MarkOpticalDuplicates) do in the reference.
func (d *DeviceSam) AddNodes(p *pipeline.Pipeline, header *sam.Header, sortingOrder sam.SortingOrder) {
	d.Header = header
	p.Add(pipeline.Seq(pipeline.Receive(func(_ int, data interface{}) interface{} {
		d.appendBatch(data.([]*sam.Alignment))
		return data
	}), pipeline.Finalize(func() {
		order := C.int(C.ELP_SO_KEEP)
		switch sortingOrder {
		case sam.Coordinate:
			order = C.ELP_SO_COORDINATE
		case sam.Queryname:
			order = C.ELP_SO_QUERYNAME
		}
		mode := C.int(0)
		if d.opts.MarkDuplicates {
			mode = C.ELP_MARKDUP
			if d.opts.AlsoOpticals {
				mode = C.ELP_MARKDUP_OPTICAL
			}
		}
		check(d.ctx, C.elp_sort_markdup(d.ctx, order, mode))
	})))
}

// RunPipeline: the source side of the write phase (sam/filter-pipeline.go:242-279): output order, FLAG and QUAL come from the device.
func (d *DeviceSam) RunPipeline(output sam.PipelineOutput, hdrFilters []sam.Filter, sortingOrder sam.SortingOrder) {
	n := uint64(C.elp_n_sorted(d.ctx)) // the output order: fewer than the reads held after FilterTargetRegions
	const chunk = uint64(1 << 18)
	idx := make([]C.uint64_t, chunk)
	flag := make([]C.uint16_t, chunk)
	off := make([]C.uint64_t, chunk+1)
	out := make([]*sam.Alignment, 0, n)
	for first := uint64(0); first < n; first += chunk {
		m := chunk
		if n-first < m {
			m = n - first
		}
		qual := make([]byte, uint64(C.elp_fetch_qual_bytes(d.ctx, C.uint64_t(first), C.uint64_t(m)))+1)
		check(d.ctx, C.elp_fetch(d.ctx, C.uint64_t(first), C.uint64_t(m), &idx[0], &flag[0], &off[0], (*C.uint8_t)(unsafe.Pointer(&qual[0])), C.uint64_t(len(qual))))
		for k := uint64(0); k < m; k++ {
			aln := d.alns[idx[k]]
			aln.FLAG = uint16(flag[k])
			aln.QUAL = qual[off[k]:off[k+1]:off[k+1]]
			out = append(out, aln)
		}
	}
	(&sam.Sam{Header: d.Header, Alignments: out}).RunPipeline(output, hdrFilters, sam.Keep)
}

// ---- operators of the path, reference names and meaning ----

// MarkOpticalDuplicates returns what filters.MarkOpticalDuplicates returns; the counting ran in the Finalize of AddNodes.
func (d *DeviceSam) MarkOpticalDuplicates() map[string]*filters.DuplicatesCtr {
	res := make(map[string]*filters.DuplicatesCtr)
	for slot := C.int32_t(0); slot < C.elp_optical_n_libraries(d.ctx); slot++ {
		var m C.elp_dup_metrics
		check(d.ctx, C.elp_optical_metrics(d.ctx, slot, &m))
		res[C.GoString(C.elp_optical_library_name(d.ctx, slot))] = &filters.DuplicatesCtr{
			UnpairedReadsExamined: int(m.unpaired_reads_examined), ReadPairsExamined: int(m.read_pairs_examined),
			SecondaryOrSupplementaryReads: int(m.secondary_or_supplementary_reads), UnmappedReads: int(m.unmapped_reads),
			UnpairedReadDuplicates: int(m.unpaired_read_duplicates), ReadPairDuplicates: int(m.read_pair_duplicates),
			ReadPairOpticalDuplicates: int(m.read_pair_optical_duplicates)}
	}
	return res
}

// PrintDuplicatesMetrics: filters.PrintDuplicatesMetrics (mark-optical-duplicates.go:601-699).
func (d *DeviceSam) PrintDuplicatesMetrics(path, commandLine, startedOn string) {
	p, c, s := C.CString(path), C.CString(commandLine), C.CString(startedOn)
	defer C.free(unsafe.Pointer(p))
	defer C.free(unsafe.Pointer(c))
	defer C.free(unsafe.Pointer(s))
	check(d.ctx, C.elp_print_duplicates_metrics(d.ctx, p, c, s))
}

// SetOutputFilter: the write-phase filters of elp_fetch_bam / elp_fetch_sam (filters2 of cmd/filter.go:803-902, and RemoveOptionalReads).
// mask: C.ELP_OUT_REMOVE_DUPLICATES (--remove-duplicates), C.ELP_OUT_REMOVE_OPTIONAL_READS (the header has @sr; drop @sr from the header
// written).  remove: the --remove-optional-fields tags; keep: the --keep-optional-fields tags, with keepFilter false for no keep filter
// ("all" / "none" are keepFilter with an empty keep).  The columnar RunPipeline above runs filters2 on the host and ignores this setting.
func (d *DeviceSam) SetOutputFilter(mask uint32, remove []string, keep []string, keepFilter bool) {
	cRemove, f1 := cstrings(remove, nil)
	cKeep, f2 := cstrings(keep, nil)
	defer f1()
	defer f2()
	if keepFilter {
		mask |= C.ELP_OUT_KEEP_FIELDS
	}
	check(d.ctx, C.elp_set_output_filter(d.ctx, C.uint32_t(mask), cRemove, C.int32_t(len(remove)), cKeep, C.int32_t(len(keep))))
}

// SetReplaceReadGroup: --replace-read-group on the byte paths (AppendBgzf, elp_append_bam / elp_append_sam, FetchBgzf and the other byte
// fetches): every read is in the one @RG of the header, and each record is written as filters.AddOrReplaceReadGroup (simple-filters.go:154-162)
// leaves it, RG:Z:id in place of its first RG field or behind its last field.  Create the DeviceSam from the header after the filter (its
// RG is []utils.StringMap{sam.ParseHeaderLineFromString(flag)}) and call this before the first append, or after a reset.  The columnar
// AddNodes path runs the reference's own filter on the host instead and does not need this call.
func (d *DeviceSam) SetReplaceReadGroup(on bool) {
	v := 0
	if on {
		v = 1
	}
	check(d.ctx, C.elp_set_replace_read_group(d.ctx, C.int(v)))
}

// The modes of SetInputDictionary (ELP_DICT_RENAME_CHROMOSOMES, ELP_DICT_REPLACE).
const (
	DictRenameChromosomes uint32 = 1
	DictReplace           uint32 = 2
)

// SetInputDictionary: --rename-chromosomes (DictRenameChromosomes) and --replace-reference-sequences (DictReplace) on the
// byte paths.  Create the DeviceSam from the header after filters.RenameChromosomes / ReplaceReferenceSequenceDictionary and pass the input
// file's @SQ as it stands in the file: the appends remap RNAME / RNEXT to the new dictionary as AddREFID would and, with REPLACE, drop the
// reads whose RNAME it lacks; FetchBgzf and the other byte fetches write the new refIDs, or the (renamed) names in SAM text.  Call it
// before the first append, or after a reset; mode 0 turns it off.  The columnar AddNodes path runs the reference's own filters instead.
func (d *DeviceSam) SetInputDictionary(mode uint32, input []utils.StringMap) {
	names := make([]string, len(input))
	lens := make([]C.int32_t, len(input)+1)
	for i, sq := range input {
		names[i] = sq["SN"]
		lens[i] = C.int32_t(sam.SQLN(sq))
	}
	cNames, free := cstrings(names, nil)
	defer free()
	check(d.ctx, C.elp_set_input_dictionary(d.ctx, C.uint32_t(mode), cNames, &lens[0], C.int32_t(len(input))))
}

// SetReference / SetKnownSites: the side inputs of filters.NewBaseRecalibrator (bqsr.go:424-443).
func (d *DeviceSam) SetReference(contig int, bases []byte) {
	check(d.ctx, C.elp_set_reference(d.ctx, C.int32_t(contig), (*C.uint8_t)(unsafe.Pointer(&bases[0])), C.uint64_t(len(bases))))
}
func (d *DeviceSam) SetKnownSites(contig int, startEnd []int32) {
	var p *C.int32_t
	if len(startEnd) > 0 {
		p = (*C.int32_t)(unsafe.Pointer(&startEnd[0]))
	}
	check(d.ctx, C.elp_set_known_sites(d.ctx, C.int32_t(contig), p, C.uint64_t(len(startEnd)/2), 0))
}

// LoadKnownSites: --known-sites as the reference takes it (cmd/filter.go:459,530-538), a list of .elsites files or VCF files (plain or
// BGZF, told apart by content, each read as vcf-to-elsites would convert it), parsed, sorted and flattened on the device into every
// contig's list.  Returns the lines whose chromosome is no @SQ SN.
func (d *DeviceSam) LoadKnownSites(paths []string) uint64 {
	cs := make([]*C.char, len(paths)+1)
	for i, p := range paths {
		cs[i] = C.CString(p)
	}
	defer func() {
		for _, c := range cs[:len(paths)] {
			C.free(unsafe.Pointer(c))
		}
	}()
	var unmatched C.uint64_t
	check(d.ctx, C.elp_load_known_sites(d.ctx, (**C.char)(unsafe.Pointer(&cs[0])), C.int32_t(len(paths)), &unmatched))
	return uint64(unmatched)
}

// LoadReference: --reference as the reference takes it (an .elfasta, fasta.OpenElfasta), or the FASTA file itself, plain or
// BGZF-compressed (fasta.ParseFasta), read and packed on the device into every contig's reference.  Returns the sequences whose name is
// no @SQ SN and the contigs left without a sequence.
func (d *DeviceSam) LoadReference(path string) (uint64, int32) {
	cp := C.CString(path)
	defer C.free(unsafe.Pointer(cp))
	var unmatched C.uint64_t
	var missing C.int32_t
	check(d.ctx, C.elp_load_reference(d.ctx, cp, &unmatched, &missing))
	return uint64(unmatched), int32(missing)
}

// Recalibrate: (*BaseRecalibrator).Recalibrate (bqsr.go:467-551).  The tables stay on the device.
// --target-regions: RemoveNonOverlappingReads(bedRegions) over the marked reads, before Recalibrate (cmd/filter.go:171-180, 288-296).
// SetTargetRegions takes one contig's BED Start / End pairs (sorted and flattened inside); FilterTargetRegions returns the reads dropped.
func (d *DeviceSam) SetTargetRegions(contig int, startEnd []int32) {
	var p *C.int32_t
	if len(startEnd) > 0 {
		p = (*C.int32_t)(unsafe.Pointer(&startEnd[0]))
	}
	check(d.ctx, C.elp_set_bqsr_target_regions(d.ctx, C.int32_t(contig), p, C.uint64_t(len(startEnd)/2), 0))
}
func (d *DeviceSam) FilterTargetRegions() uint64 {
	var removed C.uint64_t
	check(d.ctx, C.elp_filter_target_regions(d.ctx, &removed))
	return uint64(removed)
}

func (d *DeviceSam) Recalibrate() { check(d.ctx, C.elp_bqsr_gather(d.ctx)) }

// FinalizeBQSRTables + PrintBQSRTables (bqsr.go:677-694, print-bqsr.go:269-298); recalFile may be "".
func (d *DeviceSam) FinalizeAndPrintBQSRTables(recalFile string) {
	if recalFile == "" {
		check(d.ctx, C.elp_bqsr_finalize(d.ctx, nil))
		return
	}
	p := C.CString(recalFile)
	defer C.free(unsafe.Pointer(p))
	check(d.ctx, C.elp_bqsr_finalize(d.ctx, p))
}

// ApplyBQSR: (*BaseRecalibratorTables).ApplyBQSR (bqsr.go:936-1006) over all reads; RunPipeline then hands out the new QUAL.
func (d *DeviceSam) ApplyBQSR() { check(d.ctx, C.elp_bqsr_apply(d.ctx)) }

// sfm workers: --bqsr-tables-only / --bqsr-apply (cmd/filter.go:454-455, 955-997) through the .elrecal gob files.
func (d *DeviceSam) PrintBQSRTablesToIntermediateFile(name string) {
	p := C.CString(name)
	defer C.free(unsafe.Pointer(p))
	check(d.ctx, C.elp_bqsr_tables_write_elrecal(d.ctx, p))
}
func (d *DeviceSam) LoadAndCombineBQSRTables(files []string) {
	check(d.ctx, C.elp_bqsr_tables_clear(d.ctx))
	for _, f := range files {
		p := C.CString(f)
		check(d.ctx, C.elp_bqsr_tables_add_elrecal(d.ctx, p))
		C.free(unsafe.Pointer(p))
	}
}

// Several GPUs of one box: one DeviceSam per GPU (goroutine or process); id from CommUniqueID of rank 0.
func CommUniqueID() [128]byte {
	var id [128]byte
	if rc := C.elp_comm_unique_id((*C.uint8_t)(unsafe.Pointer(&id[0]))); rc != 0 {
		log.Panic("elp_comm_unique_id failed")
	}
	return id
}
func (d *DeviceSam) CommInit(id [128]byte, rank, world int, contigOwner []int32) {
	check(d.ctx, C.elp_comm_init(d.ctx, (*C.uint8_t)(unsafe.Pointer(&id[0])), C.int(rank), C.int(world)))
	check(d.ctx, C.elp_comm_set_partition(d.ctx, (*C.int32_t)(unsafe.Pointer(&contigOwner[0]))))
}
func (d *DeviceSam) AllReduceBQSRTables() { check(d.ctx, C.elp_bqsr_tables_allreduce(d.ctx)) }
func (d *DeviceSam) AllReduceMetrics()    { check(d.ctx, C.elp_optical_allreduce(d.ctx)) }
