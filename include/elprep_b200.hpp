// elprep_b200.hpp -- the host side above the C ABI in C++ (header only, C++17): elPrep's own types and operator names for the hot
// path, for callers that are compiled code like the reference (which is Go; this image has no Go toolchain, go/gpu/device_sam.go is
// the same layer as uncompiled cgo source).  Nothing here computes: it marshals sam.Alignment-shaped records into the columnar
// elp_batch, calls the library, and turns a failing return code into an exception carrying the text the reference panics with.
//
//   reference                                                       here
//   sam.Alignment (sam/sam-types.go:289-331)                        elprep::Alignment
//   sam.Header SQ / RG tables (sam/sam-types.go:60-118)             elprep::Header
//   (*sam.Sam).AddNodes receive + Finalize (filter-pipeline.go:108-128)   DeviceSam::AddNodes(batch) ... DeviceSam::Finalize(order)
//   filters.MarkDuplicates / MarkOpticalDuplicates (mark-duplicates.go:406, mark-optical-duplicates.go:468)   Options{MarkDuplicates, AlsoOpticals}, DeviceSam::MarkOpticalDuplicates()
//   (*BaseRecalibrator).Recalibrate (bqsr.go:467)                   DeviceSam::Recalibrate()
//   FinalizeBQSRTables + PrintBQSRTables (bqsr.go:677, print-bqsr.go:269)   DeviceSam::FinalizeBQSRTables(recalFile)
//   ApplyBQSR (bqsr.go:936)                                         DeviceSam::ApplyBQSR()
//   (*sam.Sam).RunPipeline as PipelineInput (filter-pipeline.go:242-279)   DeviceSam::RunPipeline(sink)
//   sam.ParseHeaderLineFromString (sam/sam-files.go:153-177)       elprep::ParseHeaderLineFromString
//   filters.AddOrReplaceReadGroup (filters/simple-filters.go:154-162)   elprep::AddOrReplaceReadGroup, DeviceSam::SetReplaceReadGroup (byte paths)
//   filters.RenameChromosomes (filters/simple-filters.go:189-204)   elprep::RenameChromosomes, DeviceSam::SetInputDictionary (byte paths)
//   filters.ReplaceReferenceSequenceDictionary (:34-60)             elprep::ReplaceReferenceSequenceDictionary, DeviceSam::SetInputDictionary (byte paths)
//   sam.MergeInputs (sam/merge-inputs.go:16-219)                   elprep::MergeInputs, DeviceSam::AddInput / SelectInput / SetTagRename (byte paths)
//   log.Panic(msg)                                                  throw elprep::Panic(msg)
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "elprep_b200.h"

namespace elprep {

struct Panic : std::runtime_error { int code; Panic(int rc, const std::string& msg) : std::runtime_error(msg), code(rc) {} };

struct CigarOperation { int32_t Length; char Operation; };           // sam/sam-types.go:675-678

// sam.Alignment with the optional fields the path reads (RG:Z, the `sr` tag of `elprep split`)
struct Alignment {
    std::string QNAME; uint16_t FLAG = 0; std::string RNAME = "*"; int32_t POS = 0; uint8_t MAPQ = 0; std::vector<CigarOperation> CIGAR;
    std::string RNEXT = "*"; int32_t PNEXT = 0, TLEN = 0;
    std::string SEQ;                   // bases as text; packed to BAM nibbles on the way in (sam-types.go:270-277: unknown characters become N)
    std::vector<uint8_t> QUAL;         // phred values without +33, one per base
    std::string RG; bool hasRG = false; bool sr = false;
};

struct Header {
    struct SQ { std::string SN; int32_t LN; };
    struct ReadGroup { std::string ID, LB, PU; bool hasLB = false, hasPU = false; };
    std::vector<SQ> sq; std::vector<ReadGroup> rg;
    std::string SO;                    // @HD SO ("" without one); ReplaceReferenceSequenceDictionary may set it to "unknown"
};

// sam.ParseHeaderLineFromString (sam/sam-files.go:153-177), the parser of `--replace-read-group`: TG:value fields separated by white space
// as strings.Fields splits them (unicode.IsSpace on the runes utf8.DecodeRuneInString decodes; a byte that is not valid UTF-8 is no space).
// Throws Panic(ELP_EINVAL) where the reference panics: a field whose third byte is not ':' (also one shorter than 3 bytes, a Go index
// panic there) and a repeated tag.
inline std::map<std::string, std::string> ParseHeaderLineFromString(const std::string& line) {
    auto rune = [&](size_t i, size_t* w) -> uint32_t {                 // (U+FFFD, 1) for an invalid byte
        const uint8_t c = (uint8_t)line[i];
        *w = 1;
        if (c < 0x80) return c;
        int n; uint8_t lo = 0x80, hi = 0xBF;
        if (c >= 0xC2 && c <= 0xDF) n = 1;
        else if (c >= 0xE0 && c <= 0xEF) { n = 2; if (c == 0xE0) lo = 0xA0; if (c == 0xED) hi = 0x9F; }
        else if (c >= 0xF0 && c <= 0xF4) { n = 3; if (c == 0xF0) lo = 0x90; if (c == 0xF4) hi = 0x8F; }
        else return 0xFFFD;
        if (i + n >= line.size()) return 0xFFFD;
        const uint8_t c1 = (uint8_t)line[i + 1];
        if (c1 < lo || c1 > hi) return 0xFFFD;
        uint32_t r = c & (n == 1 ? 0x1Fu : (n == 2 ? 0x0Fu : 0x07u));
        for (int k = 1; k <= n; k++) {
            const uint8_t ck = (uint8_t)line[i + k];
            if (ck < 0x80 || ck > 0xBF) return 0xFFFD;
            r = (r << 6) | (ck & 0x3Fu);
        }
        *w = (size_t)n + 1;
        return r;
    };
    auto space = [](uint32_t r) {                                        // unicode.IsSpace
        return r == '\t' || r == '\n' || r == '\v' || r == '\f' || r == '\r' || r == ' ' || r == 0x85 || r == 0xA0 || r == 0x1680 ||
               (r >= 0x2000 && r <= 0x200A) || r == 0x2028 || r == 0x2029 || r == 0x202F || r == 0x205F || r == 0x3000;
    };
    std::vector<std::string> fields;
    size_t start = std::string::npos;
    for (size_t i = 0, w = 1; i < line.size(); i += w) {
        if (space(rune(i, &w))) { if (start != std::string::npos) { fields.push_back(line.substr(start, i - start)); start = std::string::npos; } }
        else if (start == std::string::npos) start = i;
    }
    if (start != std::string::npos) fields.push_back(line.substr(start));
    std::map<std::string, std::string> rec;
    for (const std::string& f : fields) {
        if (f.size() < 3 || f[2] != ':') throw Panic(ELP_EINVAL, "incorrectly formatted SAM file field " + f);
        if (!rec.emplace(f.substr(0, 2), f.substr(3)).second) throw Panic(ELP_EINVAL, "duplicate field tag " + f.substr(0, 2) + " in a SAM header line");
    }
    return rec;
}

// filters.AddOrReplaceReadGroup (filters/simple-filters.go:154-162), `--replace-read-group`.  The constructor is the header part:
// header.rg becomes the one read group (an @RG without ID is ID "" without PU, so that the BQSR covariate is "" as readGroupCovariate
// returns it, filters/bqsr.go:35-51); build DeviceSam from that header.  operator() is aln.SetRG(id): apply it to every batch before
// AddNodes marshals it.  On the byte paths (AppendBgzf, FetchBgzf) call DeviceSam::SetReplaceReadGroup(true) instead.
struct AddOrReplaceReadGroup {
    std::string id;
    AddOrReplaceReadGroup(Header& header, const std::map<std::string, std::string>& readGroup) {
        Header::ReadGroup g;
        auto it = readGroup.find("ID");
        const bool hasID = it != readGroup.end();
        if (hasID) g.ID = it->second;
        if ((it = readGroup.find("LB")) != readGroup.end()) { g.LB = it->second; g.hasLB = true; }
        if (hasID && (it = readGroup.find("PU")) != readGroup.end()) { g.PU = it->second; g.hasPU = true; }
        header.rg.assign(1, g);
        id = g.ID;
    }
    void operator()(Alignment& a) const { a.RG = id; a.hasRG = true; }
    void operator()(std::vector<Alignment>& batch) const { for (Alignment& a : batch) (*this)(a); }
};

// filters.RenameChromosomes (filters/simple-filters.go:189-204), `--rename-chromosomes`.  The constructor is the header part: every @SQ SN
// becomes "chr" + SN; build DeviceSam from that header.  operator() is the AlignmentFilter: RNAME and RNEXT get the prefix unless they are
// "=" or "*"; apply it to every batch before AddNodes marshals it.  On the byte paths call DeviceSam::SetInputDictionary instead.
struct RenameChromosomes {
    explicit RenameChromosomes(Header& header) { for (Header::SQ& e : header.sq) e.SN = "chr" + e.SN; }
    bool operator()(Alignment& a) const {
        if (a.RNAME != "=" && a.RNAME != "*") a.RNAME = "chr" + a.RNAME;
        if (a.RNEXT != "=" && a.RNEXT != "*") a.RNEXT = "chr" + a.RNEXT;
        return true;
    }
};

// filters.ReplaceReferenceSequenceDictionary (filters/simple-filters.go:34-60), `--replace-reference-sequences`.  The constructor is the
// header part: with SO coordinate the SO becomes "unknown" when the new entries found in the old dictionary (utils.Find: the first match)
// do not appear in increasing old position; header.sq becomes dict.  operator() is the AlignmentFilter: a read is kept iff its RNAME is
// "*" or an SN of dict.  On the byte paths call DeviceSam::SetInputDictionary instead.
struct ReplaceReferenceSequenceDictionary {
    std::map<std::string, bool> names;
    ReplaceReferenceSequenceDictionary(Header& header, const std::vector<Header::SQ>& dict) {
        if (header.SO == "coordinate") {
            int previous = -1;
            for (const Header::SQ& e : dict) {
                int pos = -1;
                for (size_t i = 0; i < header.sq.size() && pos < 0; i++) if (header.sq[i].SN == e.SN) pos = (int)i;
                if (pos < 0) continue;
                if (pos > previous) previous = pos;
                else { header.SO = "unknown"; break; }
            }
        }
        names["*"] = true;
        for (const Header::SQ& e : dict) names[e.SN] = true;
        header.sq = dict;
    }
    bool operator()(const Alignment& a) const { return names.count(a.RNAME) != 0; }
};

// sam.Header with every line as sam.MergeInputs reads it: each record a tag -> value map
struct HeaderLines {
    using Record = std::map<std::string, std::string>;
    Record HD; std::vector<Record> SQ, RG, PG; std::vector<std::string> CO;
    std::map<std::string, std::vector<Record>> UserRecords;
};

// mergeSequenceDictionaries (sam/merge-inputs.go:100-124) as written: order-preserving and recursive.  j is set from an index in fromDict
// after a recursive merge and from an index in the new dictionary after a shared entry, so a later fromDict[j:iFrom] can start behind its
// end; Go panics on that slice, and so does this.
inline std::vector<HeaderLines::Record> MergeSequenceDictionaries(const std::vector<HeaderLines::Record>& toDict, const std::vector<HeaderLines::Record>& fromDict) {
    auto member = [](const std::vector<HeaderLines::Record>& d, const std::string& sn) -> long {   // memberOfSequenceDictionary
        for (size_t i = 0; i < d.size(); i++) { auto it = d[i].find("SN"); if (it != d[i].end() && it->second == sn) return (long)i; }
        return -1;
    };
    std::vector<HeaderLines::Record> out;
    long j = 0;
    for (size_t iTo = 0; iTo < toDict.size(); iTo++) {
        auto it = toDict[iTo].find("SN");
        const std::string sn = it == toDict[iTo].end() ? std::string() : it->second;
        const long iFrom = member(fromDict, sn);
        if (iFrom < 0) { out.push_back(toDict[iTo]); continue; }
        const long iNew = member(out, sn);
        if (iNew >= 0) {
            if (iNew != (long)iTo) throw Panic(ELP_EINVAL, "Cannot merge sequence dictionaries.");
            j = iNew + 1;
        } else {
            if (j > iFrom) throw Panic(ELP_EINVAL, "runtime error: slice bounds out of range [" + std::to_string(j) + ":" + std::to_string(iFrom) + "]");
            out = MergeSequenceDictionaries(out, std::vector<HeaderLines::Record>(fromDict.begin() + j, fromDict.begin() + iFrom));
            out.push_back(toDict[iTo]);
            j = iFrom + 1;
        }
    }
    for (size_t i = (size_t)j; i < fromDict.size(); i++) out.push_back(fromDict[i]);
    return out;
}

// sam.MergeInputs / mergeHeaders (sam/merge-inputs.go:16-219) over the parsed headers of the input files, in file order.  suffix stands for
// strconv.FormatInt(time.Now().Unix(), 10), the text a colliding @RG or @PG ID gets appended.  header: the merged header; sqMaps[k][i]: the
// merged index of input k's @SQ i (first match); rgMap / pgMap: the update filters replaceReadGroupIfExists / replaceProgramIDIfExists,
// which every record of every file runs in list order, composed into old value -> final value.  Build DeviceSam from header, then
// AddInput(input's @SQ) per file, SetTagRename("RG", rgMap) and SetTagRename("PG", pgMap).  Throws Panic where the reference panics.
struct MergedInputs {
    HeaderLines header; std::vector<std::vector<int32_t>> sqMaps; std::map<std::string, std::string> rgMap, pgMap;
};
inline MergedInputs MergeInputs(const std::vector<HeaderLines>& headers, const std::string& suffix) {
    if (headers.empty()) throw Panic(ELP_EINVAL, "MergeInputs: no input headers");
    MergedInputs m;
    HeaderLines& to = m.header;
    to = headers[0];
    struct Filter { int tag; std::string oldID, newID; };
    std::vector<Filter> filters;
    for (size_t f = 1; f < headers.size(); f++) {
        HeaderLines from = headers[f];
        for (auto& kv : from.HD) to.HD[kv.first] = kv.second;                           // mergeMetaData
        to.SQ = MergeSequenceDictionaries(to.SQ, from.SQ);
        std::map<std::string, bool> ids;                                                 // mergeReadGroups: the IDs before this file
        for (auto& r : to.RG) ids[r["ID"]] = true;
        for (auto& r : from.RG) {
            if (ids.count(r["ID"])) { const std::string old = r["ID"]; r["ID"] = old + suffix; filters.push_back({0, old, r["ID"]}); }
            to.RG.push_back(r);
        }
        std::map<std::string, bool> pgIDs; std::map<std::string, std::string> replaced;   // mergeProgramLines
        for (auto& r : to.PG) pgIDs[r["ID"]] = true;
        for (auto& r : from.PG) {
            if (pgIDs.count(r["ID"])) { const std::string old = r["ID"]; r["ID"] = old + suffix; filters.push_back({1, old, r["ID"]}); replaced[old] = r["ID"]; }
            to.PG.push_back(r);
        }
        for (size_t i = 1; i < from.RG.size(); i++) {                                   // (the PP fix-up walks the RG lines, as written)
            auto pp = to.RG[i].find("PP");
            if (pp == to.RG[i].end()) continue;
            auto nw = replaced.find(pp->second);
            if (nw != replaced.end()) pp->second = nw->second;
        }
        to.CO.insert(to.CO.end(), from.CO.begin(), from.CO.end());                       // mergeCommentLines
        for (auto& kv : from.UserRecords) to.UserRecords[kv.first] = kv.second;         // mergeUserRecords
        to.HD["SO"] = "unknown";
    }
    for (const HeaderLines& h : headers) {
        std::vector<int32_t> v;
        for (auto& s : h.SQ) {
            int32_t k = -1;
            for (size_t i = 0; i < to.SQ.size() && k < 0; i++) if (to.SQ[i].at("SN") == s.at("SN")) k = (int32_t)i;
            v.push_back(k);
        }
        m.sqMaps.push_back(v);
    }
    for (int tag = 0; tag < 2; tag++) {
        std::map<std::string, std::string>& out = tag ? m.pgMap : m.rgMap;
        for (const Filter& s : filters) {
            if (s.tag != tag || out.count(s.oldID)) continue;
            std::string v = s.oldID;
            for (const Filter& g : filters) if (g.tag == tag && v == g.oldID) v = g.newID;
            if (v != s.oldID) out[s.oldID] = v;
        }
    }
    return m;
}

enum class SortingOrder { Keep = ELP_SO_KEEP, Unknown = ELP_SO_UNKNOWN, Unsorted = ELP_SO_UNSORTED, Queryname = ELP_SO_QUERYNAME, Coordinate = ELP_SO_COORDINATE };

struct Options {                       // the `elprep filter` flags of the path (cmd/filter.go:435-481)
    int Device = 0, MaxCycle = 500, QuantizeLevels = 0; std::vector<uint8_t> SQQ; std::string TablenamePrefix = "GATK";
    int OpticalDuplicatesPixelDistance = 100; bool MarkDuplicates = false, AlsoOpticals = false;
};

struct DuplicatesCtr {                 // filters/mark-optical-duplicates.go:96-110 (the exported counters + the derived numbers)
    int64_t UnpairedReadsExamined = 0, ReadPairsExamined = 0, SecondaryOrSupplementaryReads = 0, UnmappedReads = 0, UnpairedReadDuplicates = 0,
            ReadPairDuplicates = 0, ReadPairOpticalDuplicates = 0, EstimatedLibrarySize = 0;
    double PercentDuplication = 0;
};

// the columns of one batch, exactly elp_batch's layout
struct Columns {
    std::vector<int32_t> refid, pos, nref, pnext, tlen, rg, lseq; std::vector<uint16_t> flag; std::vector<uint8_t> mapq, opt, qname, seq, qual;
    std::vector<uint64_t> qname_off{0}, cigar_off{0}; std::vector<uint32_t> cigar;
};

class DeviceSam {
  public:
    DeviceSam(const Header& header, const Options& opts) : header_(header), opts_(opts) {
        for (size_t i = 0; i < header.sq.size(); i++) refid_[header.sq[i].SN] = (int32_t)i;
        for (size_t i = 0; i < header.rg.size(); i++) rgidx_[header.rg[i].ID] = (int32_t)i;
        std::vector<const char*> names, ids, lbs, pus; std::vector<int32_t> lens;
        for (auto& s : header.sq) { names.push_back(s.SN.c_str()); lens.push_back(s.LN); }
        for (auto& g : header.rg) { ids.push_back(g.ID.c_str()); lbs.push_back(g.hasLB ? g.LB.c_str() : nullptr); pus.push_back(g.hasPU ? g.PU.c_str() : nullptr); }
        elp_config cfg; std::memset(&cfg, 0, sizeof cfg);
        cfg.device = opts.Device; cfg.n_contigs = (int32_t)header.sq.size(); cfg.contig_names = names.data(); cfg.contig_lengths = lens.data();
        cfg.n_read_groups = (int32_t)header.rg.size(); cfg.rg_id = ids.data(); cfg.rg_lb = lbs.data(); cfg.rg_pu = pus.data();
        cfg.max_cycle = opts.MaxCycle; cfg.quantize_levels = opts.QuantizeLevels; cfg.sqq = opts.SQQ.empty() ? nullptr : opts.SQQ.data(); cfg.n_sqq = (int32_t)opts.SQQ.size();
        cfg.tablename_prefix = opts.TablenamePrefix.c_str(); cfg.optical_pixel_distance = opts.OpticalDuplicatesPixelDistance;
        const int rc = elp_create(&cfg, &ctx_);
        if (rc != ELP_OK) throw Panic(rc, elp_last_error(nullptr));      // ELP_ENODEVICE included: there is no CPU path to fall back to
    }
    ~DeviceSam() { if (ctx_) elp_destroy(ctx_); }
    DeviceSam(const DeviceSam&) = delete; DeviceSam& operator=(const DeviceSam&) = delete;

    // filters.AddREFID (filters/simple-filters.go:208-231): "*" and names that are no @SQ give -1; RNEXT "=" is RNAME
    static int32_t lookup(const std::unordered_map<std::string, int32_t>& t, const std::string& name) { auto it = t.find(name); return it == t.end() ? -1 : it->second; }

    // []*sam.Alignment -> columns (what a pargo stage does per batch, sam/filter-pipeline.go:92-104).  Static: usable without a device.
    static Columns marshal(const Header& header, const std::vector<Alignment>& batch) {
        std::unordered_map<std::string, int32_t> ref, rgi;
        for (size_t i = 0; i < header.sq.size(); i++) ref[header.sq[i].SN] = (int32_t)i;
        for (size_t i = 0; i < header.rg.size(); i++) rgi[header.rg[i].ID] = (int32_t)i;
        static const char ops[] = "MIDNSHP=X", bases[] = "=ACMGRSVTWYHKDBN";
        Columns c;
        for (const Alignment& a : batch) {
            const int32_t r = lookup(ref, a.RNAME);
            c.refid.push_back(r); c.nref.push_back(a.RNEXT == "=" ? r : lookup(ref, a.RNEXT));
            c.pos.push_back(a.POS); c.pnext.push_back(a.PNEXT); c.tlen.push_back(a.TLEN); c.flag.push_back(a.FLAG); c.mapq.push_back(a.MAPQ);
            int32_t g = -1;
            if (a.hasRG) { g = lookup(rgi, a.RG); if (g < 0) throw Panic(ELP_EINVAL, "RG:Z value " + a.RG + " is not an @RG ID"); }
            c.rg.push_back(g); c.opt.push_back(a.sr ? (uint8_t)ELP_OPT_SR : (uint8_t)0);
            c.qname.insert(c.qname.end(), a.QNAME.begin(), a.QNAME.end()); c.qname_off.push_back(c.qname.size());
            for (const CigarOperation& op : a.CIGAR) {            // adjacent identical operations merge, as slowScanCigarString does (sam-types.go:700-724)
                const char* p = std::strchr(ops, op.Operation);
                if (!p || !op.Operation) throw Panic(ELP_EINVAL, std::string("unknown CIGAR operation ") + op.Operation);
                const uint32_t code = (uint32_t)(p - ops);
                if (c.cigar.size() > c.cigar_off.back() && (c.cigar.back() & 15u) == code) c.cigar.back() = (((c.cigar.back() >> 4) + (uint32_t)op.Length) << 4) | code;
                else c.cigar.push_back(((uint32_t)op.Length << 4) | code);
            }
            c.cigar_off.push_back(c.cigar.size());
            if (a.QUAL.size() != a.SEQ.size()) throw Panic(ELP_EINVAL, "QUAL must have one value per base");
            c.lseq.push_back((int32_t)a.SEQ.size());
            for (size_t i = 0; i < a.SEQ.size(); i += 2) {
                auto nib = [&](char ch) -> uint8_t { const char* p = ch ? std::strchr(bases, ch) : nullptr; return p ? (uint8_t)(p - bases) : (uint8_t)15; };
                c.seq.push_back((uint8_t)((nib(a.SEQ[i]) << 4) | (i + 1 < a.SEQ.size() ? nib(a.SEQ[i + 1]) : 0)));
            }
            c.qual.insert(c.qual.end(), a.QUAL.begin(), a.QUAL.end());
        }
        return c;
    }

    // the receive side of AddNodes: one batch of alignments, kept so that RunPipeline can hand them back in output order
    void AddNodes(const std::vector<Alignment>& batch) {
        if (batch.empty()) return;
        Columns c = marshal(header_, batch);
        static const uint8_t zero8[1] = {0}; static const uint32_t zero32[1] = {0};
        elp_batch b; std::memset(&b, 0, sizeof b);
        b.n = batch.size(); b.refid = c.refid.data(); b.pos = c.pos.data(); b.flag = c.flag.data(); b.mapq = c.mapq.data(); b.nref = c.nref.data(); b.pnext = c.pnext.data();
        b.tlen = c.tlen.data(); b.rg = c.rg.data(); b.qname_off = c.qname_off.data(); b.qname = c.qname.empty() ? zero8 : c.qname.data(); b.cigar_off = c.cigar_off.data();
        b.cigar = c.cigar.empty() ? zero32 : c.cigar.data(); b.l_seq = c.lseq.data(); b.seq = c.seq.empty() ? zero8 : c.seq.data(); b.qual = c.qual.empty() ? zero8 : c.qual.data();
        b.opt_flags = c.opt.data();
        check(elp_append_batch(ctx_, &b));
        alns_.insert(alns_.end(), batch.begin(), batch.end());
    }
    // a BGZF-compressed BAM file instead of AddNodes: its bytes in order, cut anywhere, inflated and parsed on the device (elp_append_bgzf);
    // AppendBgzfEnd after the last bytes.  RunPipeline's alignments then come from elp_fetch_bam / elp_fetch_sam, not from AddNodes.
    void AppendBgzf(const uint8_t* data, size_t n) { check(elp_append_bgzf(ctx_, data, n)); }
    void AppendBgzfEnd() { check(elp_append_bgzf_end(ctx_)); }
    // the write side: output records [first, first+n) of elp_fetch_bam behind prefix (the BAM header on a file's first call), as BGZF blocks
    // deflated on the device (elp_fetch_bgzf), with the EOF marker when eof; the bytes go to the file as they are
    std::vector<uint8_t> FetchBgzf(uint64_t first, uint64_t n, const std::vector<uint8_t>& prefix = {}, bool eof = true) {
        const uint64_t records = n ? elp_fetch_bam_bytes(ctx_, first, n) : 0;   // (0 on a refusal, which elp_fetch_bgzf then reports)
        std::vector<uint8_t> out(elp_bgzf_deflate_bound(records + prefix.size()));
        uint64_t got = 0;
        check(elp_fetch_bgzf(ctx_, first, n, prefix.empty() ? nullptr : prefix.data(), prefix.size(), eof ? 1 : 0, out.data(), out.size(), &got));
        out.resize(got);
        return out;
    }
    // --replace-read-group on the byte paths (elp_set_replace_read_group): every read of AppendBgzf is in the header's one @RG, and FetchBgzf
    // writes each record as AddOrReplaceReadGroup leaves it; before the first append (or after a reset)
    void SetReplaceReadGroup(bool on) { check(elp_set_replace_read_group(ctx_, on ? 1 : 0)); }
    // --rename-chromosomes / --replace-reference-sequences on the byte paths (elp_set_input_dictionary, mode of ELP_DICT_*): the DeviceSam
    // was built from the header after RenameChromosomes / ReplaceReferenceSequenceDictionary, input is the file's @SQ before them; AppendBgzf
    // remaps and drops as the filters do and FetchBgzf writes the new refIDs.  Before the first append (or after a reset); mode 0 turns it off
    void SetInputDictionary(uint32_t mode, const std::vector<Header::SQ>& input) {
        std::vector<const char*> names; std::vector<int32_t> lens;
        for (const Header::SQ& e : input) { names.push_back(e.SN.c_str()); lens.push_back(e.LN); }
        check(elp_set_input_dictionary(ctx_, mode, names.data(), lens.data(), (int32_t)input.size()));
    }
    // several input files on the byte paths (elp_add_input, elp_select_input, elp_set_tag_rename): the DeviceSam was built from
    // MergeInputs(...).header; AddInput once per file with its @SQ (returns its id), SelectInput before the file's AppendBgzf, and the
    // merge's rgMap / pgMap through SetTagRename.  Before the first append (or after a reset), except SelectInput
    int AddInput(const std::vector<Header::SQ>& input) {
        std::vector<const char*> names; std::vector<int32_t> lens;
        for (const Header::SQ& e : input) { names.push_back(e.SN.c_str()); lens.push_back(e.LN); }
        const int rc = elp_add_input(ctx_, names.data(), lens.data(), (int32_t)input.size());
        if (rc < 0) check(rc);
        return rc;
    }
    void SelectInput(int input) { check(elp_select_input(ctx_, input)); }
    void SetTagRename(const std::string& tag, const std::map<std::string, std::string>& map) {
        std::vector<const char*> o, n;
        for (auto& kv : map) { o.push_back(kv.first.c_str()); n.push_back(kv.second.c_str()); }
        check(elp_set_tag_rename(ctx_, tag.c_str(), o.data(), n.data(), (int32_t)o.size()));
    }
    // the Finalize of AddNodes: By(CoordinateLess / QNAMELess).ParallelStableSort + filters.MarkDuplicates (+ MarkOpticalDuplicates)
    void Finalize(SortingOrder order) { check(elp_sort_markdup(ctx_, (int)order, opts_.MarkDuplicates ? (opts_.AlsoOpticals ? ELP_MARKDUP_OPTICAL : ELP_MARKDUP) : 0)); }

    void SetReference(int contig, const std::string& bases) { check(elp_set_reference(ctx_, contig, reinterpret_cast<const uint8_t*>(bases.data()), bases.size())); }
    void SetKnownSites(int contig, const std::vector<int32_t>& startEnd) { check(elp_set_known_sites(ctx_, contig, startEnd.empty() ? nullptr : startEnd.data(), startEnd.size() / 2, 0)); }
    // --known-sites a.elsites,b.vcf.gz: every file (.elsites, or VCF plain or BGZF, told apart by content) parsed, sorted and flattened
    // on the device into every contig's list; returns the lines whose chromosome is no @SQ SN
    uint64_t LoadKnownSites(const std::vector<std::string>& paths) {
        std::vector<const char*> p;
        for (const auto& s : paths) p.push_back(s.c_str());
        uint64_t unmatched = 0;
        check(elp_load_known_sites(ctx_, p.empty() ? nullptr : p.data(), (int32_t)p.size(), &unmatched));
        return unmatched;
    }
    // --reference: an .elfasta or a FASTA file (plain or BGZF), read and packed on the device into every contig's reference; returns
    // (sequences whose name is no @SQ SN, contigs left without a sequence)
    std::pair<uint64_t, int32_t> LoadReference(const std::string& path) {
        uint64_t unmatched = 0; int32_t missing = 0;
        check(elp_load_reference(ctx_, path.c_str(), &unmatched, &missing));
        return {unmatched, missing};
    }
    // `--target-regions`: RemoveNonOverlappingReads(bedRegions) after marking, before Recalibrate (cmd/filter.go:171-180, 288-296); one
    // contig's BED Start / End pairs per call, sorted and flattened inside.  FilterTargetRegions returns the number of reads dropped.
    void SetTargetRegions(int contig, const std::vector<int32_t>& startEnd) { check(elp_set_bqsr_target_regions(ctx_, contig, startEnd.empty() ? nullptr : startEnd.data(), startEnd.size() / 2, 0)); }
    uint64_t FilterTargetRegions() { uint64_t removed = 0; check(elp_filter_target_regions(ctx_, &removed)); return removed; }
    void Recalibrate() { check(elp_bqsr_gather(ctx_)); }
    void FinalizeBQSRTables(const std::string& recalFile = "") { check(elp_bqsr_finalize(ctx_, recalFile.empty() ? nullptr : recalFile.c_str())); }
    void ApplyBQSR() { check(elp_bqsr_apply(ctx_)); }
    void PrintBQSRTablesToIntermediateFile(const std::string& name) { check(elp_bqsr_tables_write_elrecal(ctx_, name.c_str())); }
    void LoadAndCombineBQSRTables(const std::vector<std::string>& files) { check(elp_bqsr_tables_clear(ctx_)); for (auto& f : files) check(elp_bqsr_tables_add_elrecal(ctx_, f.c_str())); }

    std::map<std::string, DuplicatesCtr> MarkOpticalDuplicates() {
        std::map<std::string, DuplicatesCtr> res;
        for (int32_t slot = 0; slot < elp_optical_n_libraries(ctx_); slot++) {
            elp_dup_metrics m; check(elp_optical_metrics(ctx_, slot, &m));
            DuplicatesCtr d; d.UnpairedReadsExamined = m.unpaired_reads_examined; d.ReadPairsExamined = m.read_pairs_examined;
            d.SecondaryOrSupplementaryReads = m.secondary_or_supplementary_reads; d.UnmappedReads = m.unmapped_reads; d.UnpairedReadDuplicates = m.unpaired_read_duplicates;
            d.ReadPairDuplicates = m.read_pair_duplicates; d.ReadPairOpticalDuplicates = m.read_pair_optical_duplicates; d.EstimatedLibrarySize = m.estimated_library_size;
            d.PercentDuplication = m.percent_duplication;
            res[elp_optical_library_name(ctx_, slot)] = d;
        }
        return res;
    }
    void PrintDuplicatesMetrics(const std::string& path, const std::string& commandLine, const std::string& startedOn) {
        check(elp_print_duplicates_metrics(ctx_, path.c_str(), commandLine.c_str(), startedOn.c_str()));
    }

    // the source side of the write phase: the alignments in output order with the FLAG and QUAL the device computed
    void RunPipeline(const std::function<void(const Alignment&)>& sink, uint64_t chunk = 1u << 18) {
        const uint64_t n = elp_n_sorted(ctx_);                            // the output order: fewer than Len() after FilterTargetRegions
        std::vector<uint64_t> idx(chunk), off(chunk + 1); std::vector<uint16_t> flag(chunk); std::vector<uint8_t> qual;
        for (uint64_t first = 0; first < n; first += chunk) {
            const uint64_t m = std::min(chunk, n - first);
            qual.resize(elp_fetch_qual_bytes(ctx_, first, m) + 1);
            check(elp_fetch(ctx_, first, m, idx.data(), flag.data(), off.data(), qual.data(), qual.size()));
            for (uint64_t k = 0; k < m; k++) {
                Alignment& a = alns_[idx[k]];
                a.FLAG = flag[k]; a.QUAL.assign(qual.begin() + off[k], qual.begin() + off[k + 1]);
                sink(a);
            }
        }
    }
    uint64_t Len() const { return elp_n_reads(ctx_); }
    elp_ctx* Context() { return ctx_; }

  private:
    void check(int rc) { if (rc != ELP_OK) throw Panic(rc, elp_last_error(ctx_)); }
    elp_ctx* ctx_ = nullptr; Header header_; Options opts_; std::vector<Alignment> alns_;
    std::unordered_map<std::string, int32_t> refid_, rgidx_;
};

}  // namespace elprep
