// tagwalk.cuh -- the one statement of the BAM optional-field grammar (sam/bam-files.go:369-397) for the write-phase kernels: where a field
// ends, whether the output field filter (elp_set_output_filter) drops it, and where the RG field of --replace-read-group goes.  format_line
// (sam_format.cu) and the BAM field-filter kernels (bam_ingest.cu) walk a record's fields with out_fields; the ingest validated every record, so no bound is checked here beyond
// the record's end.  field_end is warp-collective (Z / H search their NUL with a ballot): every lane of the warp must call it with the
// same arguments.
#pragma once
#include <cstdint>
#include "common.cuh"

namespace tagwalk {

__device__ __forceinline__ uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

// first NUL at or after `from` (the ingest checked that there is one before n)
__device__ __forceinline__ uint64_t find_nul(const uint8_t* p, uint64_t from, uint64_t n) {
    const unsigned lane = threadIdx.x & 31;
    for (uint64_t b = from; b < n; b += 32) {
        const unsigned m = __ballot_sync(FULL_MASK, b + lane < n && p[b + lane] == 0);
        if (m) return b + __ffs(m) - 1;
    }
    return n;
}

// bytes per element of a B array of subtype sub (c C: 1, s S: 2, i I f: 4)
__device__ __forceinline__ int elem_size(uint8_t sub) { return (sub == 'c' || sub == 'C') ? 1 : ((sub == 's' || sub == 'S') ? 2 : 4); }

// end of the field whose tag starts at r[t] (t + 3 <= rec): tag[2] type[1] value; Z / H end behind their NUL, B is subtype, count and
// count x element size.  A type the ingest does not accept ends the walk (rec).
__device__ __forceinline__ uint64_t field_end(const uint8_t* r, uint64_t t, uint64_t rec) {
    const uint64_t v = t + 3;
    switch (r[t + 2]) {
        case 'A': case 'c': case 'C': return v + 1;
        case 's': case 'S': return v + 2;
        case 'i': case 'I': case 'f': return v + 4;
        case 'Z': case 'H': return find_nul(r, v, rec) + 1;
        case 'B': return v + 5 + (uint64_t)elem_size(r[v]) * rd32(r + v + 1);
        default: return rec;
    }
}

// the output field filter: bit (t0 | t1 << 8) of the 65 536-bit table is set when the field with tag t0 t1 is dropped
__device__ __forceinline__ bool dropped(const uint32_t* __restrict__ tab, uint8_t t0, uint8_t t1) {
    const uint32_t i = (uint32_t)t0 | ((uint32_t)t1 << 8);
    return (__ldg(tab + (i >> 5)) >> (i & 31)) & 1u;
}

// --replace-read-group (elp_set_replace_read_group): the new RG value, written as the field RG Z id NUL (n id bytes without the NUL).
// on == false: the records are written as stored.
struct RgSet { const uint8_t* id; uint32_t n; bool on; };

// The fields a record is written with, in order: aln.SetRG(id) (SmallMap.Set, utils/small-map.go:59-67) followed by the field filter
// (drop: the 65 536-bit table, or null for none).  With g.on the first field whose tag is RG, of whatever type, is replaced in place by
// the new RG:Z field and later RG fields stay as they are; a record without an RG field gets the new one behind its last field.  Then
// every field whose tag the table drops is left out, the new one included (it is tested as RG).  f(t, fe, repl) once per field written:
// repl false: the stored field r[t, fe); repl true: the new RG:Z field.  Warp-collective like field_end.
template <class F> __device__ __forceinline__ void out_fields(const uint8_t* r, uint64_t t, uint64_t rec, const uint32_t* drop, RgSet g, F f) {
    bool seen = !g.on;
    while (t + 3 <= rec) {
        const uint64_t fe = field_end(r, t, rec);
        const bool repl = !seen && r[t] == 'R' && r[t + 1] == 'G';
        seen |= repl;
        if (!drop || !dropped(drop, r[t], r[t + 1])) f(t, fe, repl);
        t = fe;
    }
    if (!seen && (!drop || !dropped(drop, 'R', 'G'))) f(rec, rec, true);
}

// the new RG:Z field's BAM bytes (3 + n + 1) at o, over the warp
__device__ __forceinline__ uint64_t rg_field_bytes(const RgSet& g) { return 4ull + g.n; }
__device__ __forceinline__ void rg_field_write(uint8_t* o, const RgSet& g) {
    const uint32_t m = g.n + 4;
    for (uint32_t j = threadIdx.x & 31; j < m; j += 32) o[j] = j == 0 ? 'R' : (j == 1 ? 'G' : (j == 2 ? 'Z' : (j < m - 1 ? g.id[j - 3] : 0)));
}

}  // namespace tagwalk

struct elp_ctx;
tagwalk::RgSet rg_set(const elp_ctx* c);   // bam_ingest.cu: the context's setting of elp_set_replace_read_group
