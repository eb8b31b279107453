/*
 * oracle/oracle.c -- TEST INFRASTRUCTURE ONLY (see oracle.h).
 *
 * Literal CPU restatement of the elPrep 5.1.3 hot path.  Structure follows the
 * reference: sharded concurrent maps + CAS "best" handles for duplicate
 * marking, a parallel stable merge sort with the full comparator, range-reduce
 * BQSR gather with per-thread tables, batch-parallel apply.  PARITY UNPINNED
 * (no reference tests/fixtures for this path; no Go toolchain here).
 *
 * Reference non-determinism fixed here (documented in DESIGN.md):
 *  - initializeCombinedBQSRTable iterates a Go map (bqsr.go:657-668): ascending qual order is used.
 *  - equal score AND equal QNAME inside one duplicate group, >2 reads sharing (LIBID,QNAME):
 *    with n_threads=1 the sequential input order decides, as a single goroutine would.
 */
#define _GNU_SOURCE
#include "oracle.h"
#include "gomath.h"
#include <pthread.h>
#include <stdatomic.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <float.h>

/* ------------------------------------------------------------------ helpers */
typedef struct { int32_t len; char op; } cigop;
static const char BAM_OPS[] = "MIDNSHP=X???????";
static inline cigop dec(uint32_t c) { cigop o; o.len = (int32_t)(c >> 4); o.op = BAM_OPS[c & 15]; return o; }
static inline uint32_t enc(cigop o) { const char *p = strchr(BAM_OPS, o.op); return ((uint32_t)o.len << 4) | (uint32_t)(p - BAM_OPS); }
static inline int consumes_read(char op) { return op == 'M' || op == 'I' || op == 'S' || op == '=' || op == 'X'; } /* sam-types.go:744 */
static inline int consumes_ref(char op) { return op == 'M' || op == 'D' || op == 'N' || op == '=' || op == 'X'; }  /* sam-types.go:746 */
static const char NIB2BASE[] = "=ACMGRSVTWYHKDBN"; /* sam-types.go:228 */
static inline char seq_base(const uint8_t *seq, int i) { uint8_t b = seq[i >> 1]; return NIB2BASE[(i & 1) ? (b & 15) : (b >> 4)]; }

typedef struct { void (*fn)(void *, int, int); void *arg; int tid, nt; } pf_task;
static void *pf_tramp(void *p) { pf_task *t = (pf_task *)p; t->fn(t->arg, t->tid, t->nt); return NULL; }
static void parallel_run(int nt, void (*fn)(void *, int, int), void *arg) {
    if (nt <= 1) { fn(arg, 0, 1); return; }
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * nt);
    pf_task *ts = (pf_task *)malloc(sizeof(pf_task) * nt);
    for (int i = 0; i < nt; i++) { ts[i].fn = fn; ts[i].arg = arg; ts[i].tid = i; ts[i].nt = nt; pthread_create(&th[i], NULL, pf_tramp, &ts[i]); }
    for (int i = 0; i < nt; i++) pthread_join(th[i], NULL);
    free(th); free(ts);
}

/* ---------------------------------------------- mark-duplicates.go:36-110 */
int32_t orc_phred_score(const uint8_t *qual, int32_t n, int *invalid) {
    /* phredScoreTable indexed by byte(char<<1): the shift wraps, so char>=128 aliases char-128 (mark-duplicates.go:38-67) */
    int32_t score = 0; int err = 0;
    for (int32_t i = 0; i < n; i++) {
        uint8_t pos = (uint8_t)(qual[i] << 1);
        int ch = pos >> 1;
        if (ch > 126 - 33) err |= 1; else if (ch >= 15) score += ch;
    }
    if (invalid) *invalid = err;
    return score;
}

int32_t orc_unclipped_position(int32_t pos, int reversed, const uint32_t *cigar, int32_t nc) {
    int32_t result = pos;
    if (nc == 0) return result;
    if (reversed) {
        int32_t clipped = 1;
        result--;
        for (int32_t i = nc - 1; i >= 0; i--) {
            cigop op = dec(cigar[i]);
            int32_t c = (op.op == 'S' || op.op == 'H');
            int32_t r = consumes_ref(op.op);
            clipped *= c;
            result += (r | clipped) * op.len;
        }
    } else {
        for (int32_t i = 0; i < nc; i++) {
            cigop op = dec(cigar[i]);
            if (!(op.op == 'S' || op.op == 'H')) break;
            result -= op.len;
        }
    }
    return result;
}

/* ---------------------------------------------- sam-types.go:408-473 */
uint16_t orc_mod_flag(uint16_t flag) {
    if ((flag & 0x1) == 0) { flag &= ~0x8; flag &= ~0x20; }
    if (flag & 0x4) flag &= ~0x10;
    if (flag & 0x8) flag &= ~0x20;
    return flag;
}

static inline int qname_cmp(const orc_reads *r, int64_t a, int64_t b) {
    uint64_t la = r->qname_off[a + 1] - r->qname_off[a], lb = r->qname_off[b + 1] - r->qname_off[b];
    uint64_t m = la < lb ? la : lb;
    int c = memcmp(r->qname + r->qname_off[a], r->qname + r->qname_off[b], m);
    if (c) return c;
    return la < lb ? -1 : (la > lb ? 1 : 0);
}

int orc_coordinate_less(const orc_reads *r, int64_t a, int64_t b) {
    int32_t refid1 = r->refid[a], refid2 = r->refid[b];
    if (refid1 < refid2) return refid1 >= 0;
    if (refid2 < refid1) return refid2 < 0;
    if (r->pos[a] < r->pos[b]) return 1;
    if (r->pos[a] > r->pos[b]) return 0;
    int rev1 = (r->flag[a] & 0x10) != 0, rev2 = (r->flag[b] & 0x10) != 0;
    if (rev1 != rev2) return !rev1;
    if (r->qname_off[a + 1] != r->qname_off[a] && r->qname_off[b + 1] != r->qname_off[b]) {
        int c = qname_cmp(r, a, b);
        if (c < 0) return 1;
        if (c > 0) return 0;
    }
    uint16_t f1 = orc_mod_flag(r->flag[a]), f2 = orc_mod_flag(r->flag[b]);
    if (f1 < f2) return 1;
    if (f1 > f2) return 0;
    if (r->mapq[a] < r->mapq[b]) return 1;
    if (r->mapq[a] > r->mapq[b]) return 0;
    if ((r->flag[a] & 1) && (r->flag[b] & 1)) {
        if (r->nref[a] < r->nref[b]) return 1; /* no special treatment of negative values */
        if (r->nref[a] > r->nref[b]) return 0;
        if (r->pnext[a] < r->pnext[b]) return 1;
        if (r->pnext[a] > r->pnext[b]) return 0;
    }
    return r->tlen[a] < r->tlen[b];
}

/* parallel stable merge sort (pargo sort.StableSort semantics: stable) */
typedef struct { const orc_reads *r; int64_t *a, *tmp; int64_t n; int nt; int64_t *bounds; } sort_ctx;
static void msort(const orc_reads *r, int64_t *a, int64_t *tmp, int64_t n) {
    if (n < 2) return;
    if (n <= 16) { /* insertion sort, stable */
        for (int64_t i = 1; i < n; i++) { int64_t v = a[i], j = i; while (j > 0 && orc_coordinate_less(r, v, a[j - 1])) { a[j] = a[j - 1]; j--; } a[j] = v; }
        return;
    }
    int64_t h = n / 2;
    msort(r, a, tmp, h); msort(r, a + h, tmp + h, n - h);
    if (!orc_coordinate_less(r, a[h], a[h - 1])) return;
    memcpy(tmp, a, sizeof(int64_t) * n);
    int64_t i = 0, j = h, k = 0;
    while (i < h && j < n) { if (orc_coordinate_less(r, tmp[j], tmp[i])) a[k++] = tmp[j++]; else a[k++] = tmp[i++]; }
    while (i < h) a[k++] = tmp[i++];
    while (j < n) a[k++] = tmp[j++];
}
static void sort_chunks(void *p, int tid, int nt) { sort_ctx *c = (sort_ctx *)p; (void)nt; int64_t lo = c->bounds[tid], hi = c->bounds[tid + 1]; msort(c->r, c->a + lo, c->tmp + lo, hi - lo); }
/* stable co-rank: number of elements taken from A among the first k outputs of merge(A,B), ties prefer A */
static int64_t corank(const orc_reads *r, int64_t k, const int64_t *A, int64_t na, const int64_t *B, int64_t nb) {
    int64_t lo = k > nb ? k - nb : 0, hi = k < na ? k : na;
    while (lo < hi) {
        int64_t i = (lo + hi) / 2, j = k - i; /* i from A, j from B */
        /* need A[i] to not belong before B[j-1]: if B[j-1] < A[i] strictly then fine; condition for i too small: A[i] <= B[j-1] i.e. !(B[j-1] < A[i]) */
        if (j > 0 && i < na && !orc_coordinate_less(r, B[j - 1], A[i])) lo = i + 1; else hi = i;
    }
    return lo;
}
typedef struct { const orc_reads *r; const int64_t *A, *B; int64_t na, nb; int64_t *out; int parts; } merge_ctx;
static void merge_part(void *p, int tid, int nt) {
    merge_ctx *c = (merge_ctx *)p; (void)nt;
    int64_t tot = c->na + c->nb;
    int64_t k0 = tot * tid / c->parts, k1 = tot * (tid + 1) / c->parts;
    int64_t i0 = corank(c->r, k0, c->A, c->na, c->B, c->nb), i1 = corank(c->r, k1, c->A, c->na, c->B, c->nb);
    int64_t j0 = k0 - i0, j1 = k1 - i1, i = i0, j = j0, k = k0;
    while (i < i1 && j < j1) { if (orc_coordinate_less(c->r, c->B[j], c->A[i])) c->out[k++] = c->B[j++]; else c->out[k++] = c->A[i++]; }
    while (i < i1) c->out[k++] = c->A[i++];
    while (j < j1) c->out[k++] = c->B[j++];
}
int orc_coordinate_sort(const orc_reads *r, int64_t *perm, int nt) {
    int64_t n = r->n;
    for (int64_t i = 0; i < n; i++) perm[i] = i;
    if (nt < 1) nt = 1;
    int64_t *tmp = (int64_t *)malloc(sizeof(int64_t) * (n > 0 ? n : 1));
    int chunks = 1; while (chunks * 2 <= nt) chunks *= 2; /* power of two */
    if (n < 4096) chunks = 1;
    int64_t *bounds = (int64_t *)malloc(sizeof(int64_t) * (chunks + 1));
    for (int i = 0; i <= chunks; i++) bounds[i] = n * i / chunks;
    sort_ctx sc = {r, perm, tmp, n, chunks, bounds};
    parallel_run(chunks, sort_chunks, &sc);
    int64_t *src = perm, *dst = tmp;
    for (int width = 1; width < chunks; width *= 2) {
        for (int c = 0; c < chunks; c += 2 * width) {
            int64_t lo = bounds[c], mid = bounds[c + width], hi = bounds[c + 2 * width];
            merge_ctx mc = {r, src + lo, src + mid, mid - lo, hi - mid, dst + lo, nt};
            parallel_run(nt, merge_part, &mc);
        }
        int64_t *t = src; src = dst; dst = t;
    }
    if (src != perm) memcpy(perm, src, sizeof(int64_t) * n);
    free(tmp); free(bounds);
    return 0;
}

/* sam/sam-types.go:479-481 + sam/filter-pipeline.go:119-123: By(QNAMELess) stable sort; perm[k] = index of k-th record */
int orc_queryname_sort(const orc_reads *r, int64_t *perm) {
    int64_t n = r->n;
    int64_t *tmp = (int64_t *)malloc(sizeof(int64_t) * (n > 0 ? n : 1));
    for (int64_t i = 0; i < n; i++) perm[i] = i;
    for (int64_t w = 1; w < n; w *= 2) {            /* bottom-up stable merge sort */
        for (int64_t lo = 0; lo < n; lo += 2 * w) {
            int64_t mid = lo + w < n ? lo + w : n, hi = lo + 2 * w < n ? lo + 2 * w : n, i = lo, j = mid, k = lo;
            while (i < mid && j < hi) { if (qname_cmp(r, perm[j], perm[i]) < 0) tmp[k++] = perm[j++]; else tmp[k++] = perm[i++]; }
            while (i < mid) tmp[k++] = perm[i++];
            while (j < hi) tmp[k++] = perm[j++];
        }
        memcpy(perm, tmp, sizeof(int64_t) * n);
    }
    free(tmp);
    return 0;
}

/* ---------------------------------------------- sharded concurrent map (pargo sync.Map semantics) */
typedef struct mnode { struct mnode *next; uint64_t hash; int64_t keyref; void *val; } mnode;
typedef struct { pthread_mutex_t mu; mnode **buckets; int64_t nb, count; mnode *freelist; char pad[24]; } mshard;
typedef int (*key_eq)(const void *ctx, int64_t stored_keyref, const void *probe);
typedef struct { mshard *shards; int ns; key_eq eq; const void *ctx; } smap;
static smap *smap_new(int splits, key_eq eq, const void *ctx) {
    smap *m = (smap *)calloc(1, sizeof(smap)); m->ns = splits; m->eq = eq; m->ctx = ctx;
    m->shards = (mshard *)calloc(splits, sizeof(mshard));
    for (int i = 0; i < splits; i++) { pthread_mutex_init(&m->shards[i].mu, NULL); m->shards[i].nb = 64; m->shards[i].buckets = (mnode **)calloc(64, sizeof(mnode *)); }
    return m;
}
static void smap_free(smap *m) {
    for (int i = 0; i < m->ns; i++) {
        mshard *s = &m->shards[i];
        for (int64_t b = 0; b < s->nb; b++) { mnode *x = s->buckets[b]; while (x) { mnode *nx = x->next; free(x); x = nx; } }
        mnode *x = s->freelist; while (x) { mnode *nx = x->next; free(x); x = nx; }
        free(s->buckets); pthread_mutex_destroy(&s->mu);
    }
    free(m->shards); free(m);
}
static inline uint64_t mix64(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33; return x; }
static void shard_grow(mshard *s) {
    int64_t nb2 = s->nb * 2; mnode **b2 = (mnode **)calloc(nb2, sizeof(mnode *));
    for (int64_t b = 0; b < s->nb; b++) { mnode *x = s->buckets[b]; while (x) { mnode *nx = x->next; int64_t k = (int64_t)((x->hash >> 20) & (uint64_t)(nb2 - 1)); x->next = b2[k]; b2[k] = x; x = nx; } }
    free(s->buckets); s->buckets = b2; s->nb = nb2;
}
/* LoadOrStore: returns existing val (found=1) or stores val (found=0) */
static void *smap_load_or_store(smap *m, uint64_t hash, const void *probe, int64_t keyref, void *val, int *found) {
    hash = mix64(hash);
    mshard *s = &m->shards[hash % (uint64_t)m->ns];
    pthread_mutex_lock(&s->mu);
    int64_t k = (int64_t)((hash >> 20) & (uint64_t)(s->nb - 1));
    for (mnode *x = s->buckets[k]; x; x = x->next) if (x->hash == hash && m->eq(m->ctx, x->keyref, probe)) { void *v = x->val; pthread_mutex_unlock(&s->mu); *found = 1; return v; }
    mnode *nn = s->freelist; if (nn) s->freelist = nn->next; else nn = (mnode *)malloc(sizeof(mnode));
    nn->hash = hash; nn->keyref = keyref; nn->val = val; nn->next = s->buckets[k]; s->buckets[k] = nn;
    if (++s->count > s->nb * 2) shard_grow(s);
    pthread_mutex_unlock(&s->mu);
    *found = 0; return val;
}
/* Load */
static void *smap_load(smap *m, uint64_t hash, const void *probe, int *found) {
    hash = mix64(hash);
    mshard *s = &m->shards[hash % (uint64_t)m->ns];
    pthread_mutex_lock(&s->mu);
    int64_t k = (int64_t)((hash >> 20) & (uint64_t)(s->nb - 1));
    for (mnode *x = s->buckets[k]; x; x = x->next) if (x->hash == hash && m->eq(m->ctx, x->keyref, probe)) { void *v = x->val; pthread_mutex_unlock(&s->mu); *found = 1; return v; }
    pthread_mutex_unlock(&s->mu);
    *found = 0; return NULL;
}
/* DeleteOrStore: if present delete and return (old,1) else store and return (_,0) */
static void *smap_delete_or_store(smap *m, uint64_t hash, const void *probe, int64_t keyref, void *val, int *deleted) {
    hash = mix64(hash);
    mshard *s = &m->shards[hash % (uint64_t)m->ns];
    pthread_mutex_lock(&s->mu);
    int64_t k = (int64_t)((hash >> 20) & (uint64_t)(s->nb - 1));
    for (mnode **px = &s->buckets[k]; *px; px = &(*px)->next) {
        mnode *x = *px;
        if (x->hash == hash && m->eq(m->ctx, x->keyref, probe)) { void *v = x->val; *px = x->next; x->next = s->freelist; s->freelist = x; s->count--; pthread_mutex_unlock(&s->mu); *deleted = 1; return v; }
    }
    mnode *nn = s->freelist; if (nn) s->freelist = nn->next; else nn = (mnode *)malloc(sizeof(mnode));
    nn->hash = hash; nn->keyref = keyref; nn->val = val; nn->next = s->buckets[k]; s->buckets[k] = nn;
    if (++s->count > s->nb * 2) shard_grow(s);
    pthread_mutex_unlock(&s->mu);
    *deleted = 0; return NULL;
}

/* ---------------------------------------------- mark-duplicates.go:112-445 */
typedef struct { int32_t lb, refid, pos; int reversed; } fragment_key;               /* :188-193 */
typedef struct { int32_t lb; int64_t aln; } pairfrag_key;                             /* :257-260 (qname via aln) */
typedef struct { int32_t lb, refid1, refid2; int64_t pos; int rev1, rev2; } pair_key; /* :271-276 */
typedef struct ocons { int64_t aln; struct ocons *next; } ocons;                        /* alnCons :303-306 */
typedef struct { int32_t score; int64_t aln1, aln2; pair_key key; ocons *optical; } aln_pair; /* :285-289 */
typedef struct { _Atomic(int64_t) object; } frag_handle;                              /* :160-174, object = aln index */
typedef struct { _Atomic(aln_pair *) object; pair_key key; } pair_handle;
typedef struct blk { struct blk *next; size_t used; char data[1 << 20]; } blk;
typedef struct { blk *head; } arena;
static void *arena_alloc(arena *a, size_t sz) {
    sz = (sz + 15) & ~(size_t)15;
    if (!a->head || a->head->used + sz > sizeof(a->head->data)) { blk *b = (blk *)malloc(sizeof(blk)); b->next = a->head; b->used = 0; a->head = b; }
    void *p = a->head->data + a->head->used; a->head->used += sz; return p;
}
static void arena_free(arena *a) { blk *b = a->head; while (b) { blk *n = b->next; free(b); b = n; } a->head = NULL; }

typedef struct {
    const orc_reads *r; const orc_header *h;
    int32_t *upos, *score, *lib;
    smap *fragments, *pairs_fragments, *pairs;
    frag_handle *frag_handles_unused;
    _Atomic(int64_t) next_batch; _Atomic(int) invalid;
    arena *arenas; int n_arenas;
} md_ctx;

static int frag_eq(const void *ctx, int64_t kr, const void *probe) {
    const md_ctx *c = (const md_ctx *)ctx; const fragment_key *p = (const fragment_key *)probe;
    return c->lib[kr] == p->lb && c->r->refid[kr] == p->refid && c->upos[kr] == p->pos && (((c->r->flag[kr] & 0x10) != 0) == p->reversed);
}
static int pairfrag_eq(const void *ctx, int64_t kr, const void *probe) {
    const md_ctx *c = (const md_ctx *)ctx; const pairfrag_key *p = (const pairfrag_key *)probe;
    return c->lib[kr] == p->lb && qname_cmp(c->r, kr, p->aln) == 0;
}
static int pair_eq(const void *ctx, int64_t kr, const void *probe) {
    (void)ctx; const pair_key *a = &((const pair_handle *)(intptr_t)kr)->key, *p = (const pair_key *)probe;
    return a->lb == p->lb && a->refid1 == p->refid1 && a->refid2 == p->refid2 && a->pos == p->pos && a->rev1 == p->rev1 && a->rev2 == p->rev2;
}
static inline void set_dup(const orc_reads *r, int64_t i) { __atomic_fetch_or(&r->flag[i], (uint16_t)0x400, __ATOMIC_RELAXED); }
static inline int is_true_pair(uint16_t f) { return (f & (0x1 | 0x8)) == 0x1; }     /* :182-184 */
static inline int is_true_fragment(uint16_t f) { return (f & (0x1 | 0x8)) != 0x1; } /* :177-179 */
static uint64_t qname_hash(const orc_reads *r, int64_t i) { /* DJBX33A-like; value only shards the map */
    uint64_t h = 5381; for (uint64_t k = r->qname_off[i]; k < r->qname_off[i + 1]; k++) h = h * 33 + r->qname[k]; return h;
}

static void classify_fragment(md_ctx *c, int64_t aln, arena *ar) { /* :210-254 */
    const orc_reads *r = c->r;
    fragment_key k = {c->lib[aln], r->refid[aln], c->upos[aln], (r->flag[aln] & 0x10) != 0};
    frag_handle *nh = (frag_handle *)arena_alloc(ar, sizeof(frag_handle)); atomic_init(&nh->object, aln);
    int found;
    uint64_t hash = (uint64_t)(uint32_t)k.lb * 0x9E3779B97F4A7C15ULL ^ (uint64_t)(uint32_t)k.refid ^ ((uint64_t)(uint32_t)k.pos << 20) ^ (uint64_t)k.reversed;
    frag_handle *best = (frag_handle *)smap_load_or_store(c->fragments, hash, &k, aln, nh, &found);
    if (!found) return;
    uint16_t aflag = __atomic_load_n(&r->flag[aln], __ATOMIC_RELAXED);
    if (is_true_fragment(aflag)) {
        int32_t aln_score = c->score[aln];
        for (;;) {
            int64_t best_aln = atomic_load(&best->object);
            if (is_true_pair(r->flag[best_aln])) { set_dup(r, aln); break; }
            int32_t best_score = c->score[best_aln];
            if (best_score > aln_score) { set_dup(r, aln); break; }
            else if (best_score == aln_score) {
                if (qname_cmp(r, aln, best_aln) > 0) { set_dup(r, aln); break; }
                else if (atomic_compare_exchange_strong(&best->object, &best_aln, aln)) { set_dup(r, best_aln); break; }
            } else if (atomic_compare_exchange_strong(&best->object, &best_aln, aln)) { set_dup(r, best_aln); break; }
        }
    } else {
        for (;;) {
            int64_t best_aln = atomic_load(&best->object);
            if (is_true_pair(r->flag[best_aln])) break;
            else if (atomic_compare_exchange_strong(&best->object, &best_aln, aln)) { set_dup(r, best_aln); break; }
        }
    }
}

static void classify_pair(md_ctx *c, int64_t aln, arena *ar) { /* :329-396 */
    const orc_reads *r = c->r;
    if (!is_true_pair(r->flag[aln])) return;
    int64_t aln1 = aln, aln2;
    pairfrag_key pk = {c->lib[aln], aln};
    int deleted;
    void *entry = smap_delete_or_store(c->pairs_fragments, (uint64_t)(uint32_t)c->lib[aln] * 31 ^ qname_hash(r, aln), &pk, aln, (void *)(intptr_t)(aln + 1), &deleted);
    if (!deleted) return;
    aln2 = (int64_t)(intptr_t)entry - 1;
    int32_t score = c->score[aln1] + c->score[aln2];
    int32_t refid1 = r->refid[aln1], refid2 = r->refid[aln2];
    int32_t pos1 = c->upos[aln1], pos2 = c->upos[aln2];
    int rev1 = (r->flag[aln1] & 0x10) != 0, rev2 = (r->flag[aln2] & 0x10) != 0;
    if (refid1 > refid2 || (refid1 == refid2 && (pos1 > pos2 || (pos1 == pos2 && rev1 && !rev2)))) {
        int64_t t = aln1; aln1 = aln2; aln2 = t;
        int32_t t32 = refid1; refid1 = refid2; refid2 = t32;
        t32 = pos1; pos1 = pos2; pos2 = t32;
        rev1 = (r->flag[aln1] & 0x10) != 0; rev2 = (r->flag[aln2] & 0x10) != 0;
    }
    pair_key key = {c->lib[aln1], refid1, refid2, (int64_t)((uint64_t)(int64_t)pos1 << 32) + (int64_t)pos2, rev1, rev2};
    aln_pair *np = (aln_pair *)arena_alloc(ar, sizeof(aln_pair)); np->score = score; np->aln1 = aln1; np->aln2 = aln2; np->key = key; np->optical = NULL;
    pair_handle *nh = (pair_handle *)arena_alloc(ar, sizeof(pair_handle)); atomic_init(&nh->object, np); nh->key = key;
    int found;
    uint64_t hash = (uint64_t)(uint32_t)key.lb * 0x9E3779B97F4A7C15ULL ^ (uint64_t)(uint32_t)refid1 ^ ((uint64_t)(uint32_t)refid2 << 7) ^ (uint64_t)key.pos ^ ((uint64_t)rev1 << 62) ^ ((uint64_t)rev2 << 63);
    pair_handle *best = (pair_handle *)smap_load_or_store(c->pairs, hash, &key, (int64_t)(intptr_t)nh, nh, &found);
    if (!found) return;
    for (;;) {
        aln_pair *bp = atomic_load(&best->object);
        if (bp->score > score) { set_dup(r, aln1); set_dup(r, aln2); break; }
        else if (bp->score == score) {
            if (qname_cmp(r, aln1, bp->aln1) > 0) { set_dup(r, aln1); set_dup(r, aln2); break; }
            else if (atomic_compare_exchange_strong(&best->object, &bp, np)) { set_dup(r, bp->aln1); set_dup(r, bp->aln2); break; }
        } else if (atomic_compare_exchange_strong(&best->object, &bp, np)) { set_dup(r, bp->aln1); set_dup(r, bp->aln2); break; }
    }
}

#define MD_BATCH 4096
static void md_worker(void *p, int tid, int nt) {
    md_ctx *c = (md_ctx *)p; (void)nt;
    const orc_reads *r = c->r; arena *ar = &c->arenas[tid];
    for (;;) {
        int64_t b = atomic_fetch_add(&c->next_batch, 1);
        int64_t lo = b * MD_BATCH, hi = lo + MD_BATCH; if (lo >= r->n) break; if (hi > r->n) hi = r->n;
        for (int64_t i = lo; i < hi; i++) {
            if ((r->flag[i] & (0x4 | 0x100 | 0x800)) != 0) continue; /* :436 */
            /* addLIBID :142-150 */
            c->lib[i] = (r->rg[i] >= 0 && r->rg[i] < c->h->n_rg) ? c->h->rg_lib[r->rg[i]] : -1;
            /* adaptAlignment :153-156 */
            c->upos[i] = orc_unclipped_position(r->pos[i], (r->flag[i] & 0x10) != 0, r->cigar + r->cigar_off[i], (int32_t)(r->cigar_off[i + 1] - r->cigar_off[i]));
            int inv; c->score[i] = orc_phred_score(r->qual + r->qual_off[i], r->lseq[i], &inv);
            if (inv) { atomic_store(&c->invalid, 1); continue; }
            classify_fragment(c, i, ar);
            classify_pair(c, i, ar);
        }
    }
}

static void md_init(md_ctx *c, const orc_reads *r, const orc_header *h, int nt) {
    memset(c, 0, sizeof(*c)); c->r = r; c->h = h;
    int64_t n = r->n > 0 ? r->n : 1;
    c->upos = (int32_t *)calloc(n, 4); c->score = (int32_t *)calloc(n, 4); c->lib = (int32_t *)malloc(n * 4);
    for (int64_t i = 0; i < r->n; i++) c->lib[i] = -1;
    int splits = 16 * nt; /* :407 */
    c->fragments = smap_new(splits, frag_eq, c); c->pairs_fragments = smap_new(splits, pairfrag_eq, c); c->pairs = smap_new(splits, pair_eq, c);
    c->arenas = (arena *)calloc(nt, sizeof(arena)); c->n_arenas = nt;
    atomic_init(&c->next_batch, 0); atomic_init(&c->invalid, 0);
}
static void md_free(md_ctx *c) {
    smap_free(c->fragments); smap_free(c->pairs_fragments); smap_free(c->pairs);
    for (int i = 0; i < c->n_arenas; i++) arena_free(&c->arenas[i]);
    free(c->arenas); free(c->upos); free(c->score); free(c->lib);
}

int orc_mark_duplicates(const orc_reads *r, const orc_header *h, int nt, int32_t *upos_out, int32_t *score_out) {
    if (nt < 1) nt = 1;
    md_ctx c; md_init(&c, r, h, nt);
    parallel_run(nt, md_worker, &c);
    if (upos_out) memcpy(upos_out, c.upos, r->n * 4);
    if (score_out) memcpy(score_out, c.score, r->n * 4);
    int inv = atomic_load(&c.invalid);
    md_free(&c);
    return inv ? -1 : 0;
}

/* ---------------------------------------------- filters/mark-optical-duplicates.go (+ graph.go, unpedantic.go:32-34) */
typedef struct { int64_t t, x, y; } tile_info;
/* strconv.ParseInt(s, 10, 64) as internal.ParseInt uses it (internal/strconv.go:27-33): optional sign, digits only */
static int parse_int64(const uint8_t *s, int64_t n, int64_t *out) {
    int64_t i = 0; int neg = 0;
    if (n > 0 && (s[0] == '+' || s[0] == '-')) { neg = s[0] == '-'; i = 1; }
    if (i >= n) return -1;
    uint64_t v = 0, lim = neg ? (uint64_t)1 << 63 : ((uint64_t)1 << 63) - 1;
    for (; i < n; i++) {
        if (s[i] < '0' || s[i] > '9') return -1;
        uint64_t d = (uint64_t)(s[i] - '0');
        if (v > (lim - d) / 10) return -1; /* value out of range */
        v = v * 10 + d;
    }
    *out = neg ? (int64_t)(0 - v) : (int64_t)v;
    return 0;
}
/* computeTileInfo :50-71. returns -1 where the reference panics (a field that does not parse) */
static int compute_tile_info(const orc_reads *r, int64_t aln, tile_info *ti) {
    const uint8_t *q = r->qname + r->qname_off[aln]; int64_t n = (int64_t)(r->qname_off[aln + 1] - r->qname_off[aln]);
    int64_t start[8], end[8]; int nc = 0; int64_t b = 0;
    for (int64_t i = 0; i <= n; i++) if (i == n || q[i] == ':') { if (nc < 8) { start[nc] = b; end[nc] = i; } nc++; b = i + 1; }
    int f0;
    if (nc == 7) f0 = 4; else if (nc == 5) f0 = 2; else { ti->t = ti->x = ti->y = -1; return 0; }
    if (parse_int64(q + start[f0], end[f0] - start[f0], &ti->t)) return -1;
    if (parse_int64(q + start[f0 + 1], end[f0 + 1] - start[f0 + 1], &ti->x)) return -1;
    if (parse_int64(q + start[f0 + 2], end[f0 + 2] - start[f0 + 2], &ti->y)) return -1;
    return 0;
}
static inline int64_t abs64(int64_t v) { return v < 0 ? -v : v; }
static int optical_short(const tile_info *a, const tile_info *b, int d) { return abs64(a->x - b->x) <= d && abs64(a->y - b->y) <= d; } /* unpedantic.go:32-34 */
static int optical_full(const orc_reads *r, int64_t a1, const tile_info *t1, int64_t a2, const tile_info *t2, int d) { /* :82-93 */
    if (r->rg[a1] != r->rg[a2]) return 0;
    if (t1->t == -1 || t2->t == -1) return 0;
    if (t1->t != t2->t) return 0;
    return optical_short(t1, t2, d);
}
static int64_t uf_find(int64_t *g, int64_t x) { int64_t rep = x; while (rep != g[rep]) rep = g[rep]; while (x != rep) { int64_t nx = g[x]; g[x] = rep; x = nx; } return rep; } /* graph.go:49-60 */
/* countOpticalDuplicatesFromSlice :329-373 (+ countOpticalDuplicatesWithGraph :244-273). *err set where the reference panics */
static int64_t count_optical_from_slice(const orc_reads *r, const int64_t *dups, int64_t n, int d, int *err) {
    if (n > 300000) return 0;
    if (n < 2) return 0;
    tile_info *ti = (tile_info *)malloc(sizeof(tile_info) * n);
    for (int64_t i = 0; i < n; i++) if (compute_tile_info(r, dups[i], &ti[i])) { *err = 1; free(ti); return 0; }
    int64_t ctr = 0;
    if (n >= 4) {
        /* edges inside each (RG, tile) group with tile != -1; Σ(cluster size - 1) = n - number of clusters */
        int64_t *g = (int64_t *)malloc(sizeof(int64_t) * n);
        for (int64_t i = 0; i < n; i++) g[i] = i;
        for (int64_t i = 0; i < n; i++) {
            if (ti[i].t == -1) continue;
            for (int64_t j = i + 1; j < n; j++) {
                if (ti[j].t != ti[i].t || r->rg[dups[i]] != r->rg[dups[j]]) continue;
                if (optical_short(&ti[i], &ti[j], d)) { int64_t a = uf_find(g, j), b = uf_find(g, i); if (a != b) g[a] = b; }
            }
        }
        int64_t clusters = 0;
        for (int64_t i = 0; i < n; i++) if (uf_find(g, i) == i) clusters++;
        ctr = n - clusters;
        free(g);
    } else {
        if (optical_full(r, dups[0], &ti[0], dups[1], &ti[1], d)) ctr++;
        if (n >= 3) {
            if (optical_full(r, dups[0], &ti[0], dups[2], &ti[2], d)) ctr++;
            if (ctr != 2 && optical_full(r, dups[1], &ti[1], dups[2], &ti[2], d)) ctr++;
        }
    }
    free(ti);
    return ctr;
}

typedef struct { int64_t *v; int64_t cap; } ohist;
static void ohist_inc(ohist *h, int64_t idx) {
    if (idx >= h->cap) { int64_t nc = h->cap ? h->cap : 64; while (nc <= idx) nc *= 2; h->v = (int64_t *)realloc(h->v, sizeof(int64_t) * nc); memset(h->v + h->cap, 0, sizeof(int64_t) * (nc - h->cap)); h->cap = nc; }
    h->v[idx]++;
}
struct orc_optical_result { int slots; orc_dup_metrics *m; ohist *hist; /* [slots][3]: all, non-optical, optical */ int error; };

/* estimateLibrarySize :533-562 */
static int64_t estimate_library_size(int64_t n_pairs, int64_t n_unique) {
    double n = (double)n_pairs, c = (double)n_unique;
    if (n_pairs > 0 && n_pairs - n_unique > 0) {
        double m = 1.0, M = 100.0;
#define OF(x) (c / (x)-1 + gm_exp(-n / (x)))
        double fd = OF(M * c);
        while (fd >= 0.0) { M *= 10.0; fd = OF(M * c); }
        for (int i = 0; i < 40; i++) {
            double rr = (m + M) / 2.0, u = OF(rr * c);
            if (u == 0.0) break;
            if (u > 0.0) m = rr;
            if (u < 0.0) M = rr;
        }
#undef OF
        return (int64_t)(c * ((m + M) / 2.0));
    }
    return 0;
}
/* calculateDerivedDuplicateMetrics :519-525, estimateRoi :570-572, histogramRoi :574-581 */
void orc_derive_dup_metrics(orc_dup_metrics *m) {
    m->has_roi = 0; m->estimated_library_size = 0;
    if (m->read_pairs_examined > 0) {
        m->estimated_library_size = estimate_library_size(m->read_pairs_examined - m->read_pair_optical_duplicates, m->read_pairs_examined - m->read_pair_duplicates);
        int64_t uniq = m->read_pairs_examined - m->read_pair_duplicates;
        for (int64_t x = 1; x <= 100; x++)
            m->roi[x - 1] = (double)m->estimated_library_size * (1.0 - gm_exp(-(double)(x * m->read_pairs_examined) / (double)m->estimated_library_size)) / (double)uniq;
        m->has_roi = 1;
    }
    m->percent_duplication = (double)(m->unpaired_read_duplicates + m->read_pair_duplicates * 2) / (double)(m->unpaired_reads_examined + m->read_pairs_examined * 2);
}

/* MarkDuplicates(alsoOpticals=true) followed by MarkOpticalDuplicates (:468-517) over the reads taken in `order`
 * (the sorted order in the reference; NULL = as given). Sequential. */
orc_optical_result *orc_markdup_optical(const orc_reads *r, const orc_header *h, int nt, const int64_t *order, int pixel_distance) {
    if (nt < 1) nt = 1;
    md_ctx c; md_init(&c, r, h, nt);
    parallel_run(nt, md_worker, &c);
    orc_optical_result *res = (orc_optical_result *)calloc(1, sizeof(*res));
    int n_lib = 0; for (int i = 0; i < h->n_rg; i++) if (h->rg_lib[i] + 1 > n_lib) n_lib = h->rg_lib[i] + 1;
    res->slots = n_lib + 1; res->m = (orc_dup_metrics *)calloc(res->slots, sizeof(orc_dup_metrics)); res->hist = (ohist *)calloc((size_t)res->slots * 3, sizeof(ohist));
    if (atomic_load(&c.invalid)) { res->error = -1; md_free(&c); return res; }
    /* addLIBID for all reads (:426) */
    for (int64_t i = 0; i < r->n; i++) c.lib[i] = (r->rg[i] >= 0 && r->rg[i] < h->n_rg) ? h->rg_lib[r->rg[i]] : -1;
    arena *ar = &c.arenas[0];
    smap *pf = smap_new(16, pairfrag_eq, &c);
    for (int64_t k = 0; k < r->n && !res->error; k++) {
        int64_t aln = order ? order[k] : k;
        orc_dup_metrics *ctr = &res->m[c.lib[aln] + 1];
        uint16_t f = r->flag[aln];
        if (f & 0x4) { ctr->unmapped_reads++; continue; }
        if (f & (0x100 | 0x800)) { ctr->secondary_or_supplementary++; continue; }
        if (is_true_fragment(f)) ctr->unpaired_reads_examined++;
        if (is_true_pair(f)) ctr->read_pairs_examined++;
        if (!(f & 0x400)) continue;
        if (is_true_fragment(f)) ctr->unpaired_read_duplicates++;          /* markOpticalDuplicatesFragment :176-180 */
        if (!is_true_pair(f)) continue;                                     /* markOpticalDuplicatesPair :182-224 */
        pairfrag_key pk = {c.lib[aln], aln}; int deleted;
        void *entry = smap_delete_or_store(pf, (uint64_t)(uint32_t)c.lib[aln] * 31 ^ qname_hash(r, aln), &pk, aln, (void *)(intptr_t)(aln + 1), &deleted);
        if (!deleted) continue;
        int64_t aln1 = aln, aln2 = (int64_t)(intptr_t)entry - 1;
        ctr->read_pair_duplicates++;
        int32_t refid1 = r->refid[aln1], refid2 = r->refid[aln2], pos1 = c.upos[aln1], pos2 = c.upos[aln2];
        int rev1 = (r->flag[aln1] & 0x10) != 0, rev2 = (r->flag[aln2] & 0x10) != 0;
        if (refid1 > refid2 || (refid1 == refid2 && (pos1 > pos2 || (pos1 == pos2 && rev1 && !rev2)))) {
            int64_t t = aln1; aln1 = aln2; aln2 = t; int32_t t32 = refid1; refid1 = refid2; refid2 = t32; t32 = pos1; pos1 = pos2; pos2 = t32;
            rev1 = (r->flag[aln1] & 0x10) != 0; rev2 = (r->flag[aln2] & 0x10) != 0;
        }
        pair_key key = {c.lib[aln1], refid1, refid2, (int64_t)((uint64_t)(int64_t)pos1 << 32) + (int64_t)pos2, rev1, rev2};
        uint64_t hash = (uint64_t)(uint32_t)key.lb * 0x9E3779B97F4A7C15ULL ^ (uint64_t)(uint32_t)refid1 ^ ((uint64_t)(uint32_t)refid2 << 7) ^ (uint64_t)key.pos ^ ((uint64_t)rev1 << 62) ^ ((uint64_t)rev2 << 63);
        int found;
        pair_handle *best = (pair_handle *)smap_load(c.pairs, hash, &key, &found);
        if (!found || !best) { res->error = -2; break; }                    /* "origin for duplicate read pair unknown" :210 */
        aln_pair *bp = atomic_load(&best->object);
        if (bp->aln1 != aln1) {
            ocons *e = (ocons *)arena_alloc(ar, sizeof(ocons));
            e->aln = (r->flag[aln1] & 0x40) ? aln1 : aln2;                  /* :216-221 */
            e->next = bp->optical; bp->optical = e;
        }
    }
    for (int i = 0; i < res->slots; i++) res->m[i].read_pairs_examined /= 2;  /* :503-505 */
    /* countOpticalDuplicatesPairs :380-431 over every entry of the pairs map */
    int64_t *fwd = NULL, *rev = NULL; int64_t capf = 0, capr = 0;
    for (int si = 0; si < c.pairs->ns && !res->error; si++) {
        mshard *s = &c.pairs->shards[si];
        for (int64_t b = 0; b < s->nb && !res->error; b++) for (mnode *x = s->buckets[b]; x; x = x->next) {
            aln_pair *origin = atomic_load(&((pair_handle *)x->val)->object);
            int64_t nf = 0, nr = 0;
            int64_t oaln = (r->flag[origin->aln1] & 0x40) ? origin->aln1 : origin->aln2;   /* countOpticalDuplicates :275-327 */
#define PUSH(arr, nn, cap, v) do { if (nn >= cap) { cap = cap ? cap * 2 : 64; arr = (int64_t *)realloc(arr, sizeof(int64_t) * cap); } arr[nn++] = (v); } while (0)
            if (r->flag[oaln] & 0x10) PUSH(rev, nr, capr, oaln); else PUSH(fwd, nf, capf, oaln);
            for (ocons *e = origin->optical; e; e = e->next) {
                if (r->flag[e->aln] & 0x10) { if (nr <= 300000) PUSH(rev, nr, capr, e->aln); }
                else { if (nf <= 300000) PUSH(fwd, nf, capf, e->aln); }
            }
#undef PUSH
            int err = 0;
            int64_t fc = count_optical_from_slice(r, fwd, nf, pixel_distance, &err), rc = count_optical_from_slice(r, rev, nr, pixel_distance, &err);
            if (err) { res->error = -3; break; }
            int64_t optical = fc + rc, dupcount = nf + nr;
            int slot = c.lib[origin->aln1] + 1;
            res->m[slot].read_pair_optical_duplicates += optical;
            ohist *hh = &res->hist[(size_t)slot * 3];
            ohist_inc(&hh[0], dupcount);                                    /* incrementDuplicatesCountsHistograms :150-174 */
            if (dupcount - optical > 0) ohist_inc(&hh[1], dupcount - optical);
            if (optical > 0) ohist_inc(&hh[2], optical + 1);
        }
    }
    free(fwd); free(rev);
    for (int i = 0; i < res->slots; i++) orc_derive_dup_metrics(&res->m[i]);
    smap_free(pf);
    md_free(&c);
    return res;
}
int orc_optical_error(const orc_optical_result *res) { return res->error; }
int orc_optical_slots(const orc_optical_result *res) { return res->slots; }
void orc_optical_get(const orc_optical_result *res, int slot, orc_dup_metrics *out) { *out = res->m[slot]; }
int64_t orc_optical_hist(const orc_optical_result *res, int slot, int which, int64_t *keys, int64_t *counts, int64_t cap) {
    const ohist *h = &res->hist[(size_t)slot * 3 + which]; int64_t n = 0;
    for (int64_t i = 0; i < h->cap; i++) if (h->v[i]) { if (n < cap) { keys[n] = i; counts[n] = h->v[i]; } n++; }
    return n;
}
void orc_optical_free(orc_optical_result *res) {
    if (!res) return;
    for (int i = 0; i < res->slots * 3; i++) free(res->hist[i].v);
    free(res->hist); free(res->m); free(res);
}
/* formatFloat :583-599 */
static void format_float(double f, char *out) {
    if (f != f) { strcpy(out, "NaN"); return; }
    sprintf(out, "%.6f", f);
    char *dot = strchr(out, '.'); if (!dot) return;
    for (char *j = out + strlen(out) - 1; j > dot; j--) if (*j != '0') { j[1] = 0; return; }
}
/* PrintDuplicatesMetrics :601-699. Go iterates its map in random order; here: libraries in ascending name order
 * ("Unknown Library" = slot 0 takes its place by name). lib_names[slots-1]. */
int orc_optical_print(const orc_optical_result *res, const char *const *lib_names, const char *path, const char *command_line, const char *started_on) {
    FILE *f = fopen(path, "w"); if (!f) return -1;
    int n = res->slots; int *ord = (int *)malloc(sizeof(int) * n); const char **nm = (const char **)malloc(sizeof(char *) * n);
    for (int i = 0; i < n; i++) { ord[i] = i; nm[i] = i == 0 ? "Unknown Library" : lib_names[i - 1]; }
    for (int i = 1; i < n; i++) for (int j = i; j > 0 && strcmp(nm[ord[j]], nm[ord[j - 1]]) < 0; j--) { int t = ord[j]; ord[j] = ord[j - 1]; ord[j - 1] = t; }
    fprintf(f, "## htsjdk.samtools.metrics.StringHeader\n# %s\n## htsjdk.samtools.metrics.StringHeader\n# Started on: %s\n\n## METRICS CLASS\tpicard.sam.DuplicationMetrics\n", command_line, started_on);
    fprintf(f, "LIBRARY\tUNPAIRED_READS_EXAMINED\tREAD_PAIRS_EXAMINED\tSECONDARY_OR_SUPPLEMENTARY_RDS\tUNMAPPED_READS\tUNPAIRED_READ_DUPLICATES\tREAD_PAIR_DUPLICATES\tREAD_PAIR_OPTICAL_DUPLICATES\tPERCENT_DUPLICATION\tESTIMATED_LIBRARY_SIZE\n");
    char buf[64]; int the = -1, many = 0;
    for (int k = 0; k < n; k++) {
        const orc_dup_metrics *m = &res->m[ord[k]];
        format_float(m->percent_duplication, buf);
        fprintf(f, "%s\t%lld\t%lld\t%lld\t%lld\t%lld\t%lld\t%lld\t%s", nm[ord[k]], (long long)m->unpaired_reads_examined, (long long)m->read_pairs_examined, (long long)m->secondary_or_supplementary,
                (long long)m->unmapped_reads, (long long)m->unpaired_read_duplicates, (long long)m->read_pair_duplicates, (long long)m->read_pair_optical_duplicates, buf);
        if (m->read_pairs_examined > 0) { fprintf(f, "\t%lld", (long long)m->estimated_library_size); if (the >= 0) many = 1; the = ord[k]; }
        fprintf(f, "\n");
    }
    fprintf(f, "\n");
    if (many || the < 0) { fprintf(f, "\n"); fclose(f); free(ord); free(nm); return 0; }
    const orc_dup_metrics *m = &res->m[the]; const ohist *hh = &res->hist[(size_t)the * 3];
#define HV(w, k) ((k) < hh[w].cap ? (long long)hh[w].v[k] : 0LL)
    fprintf(f, "## HISTOGRAM\tjava.lang.Double\nBIN\tCoverageMult\tall_sets\toptical_sets\tnon_optical_sets\n");
    for (int i = 0; i < 100; i++) { format_float(m->roi[i], buf); fprintf(f, "%d.0\t%s\t%lld\t%lld\t%lld\n", i + 1, buf, HV(0, i + 1), HV(2, i + 1), HV(1, i + 1)); }
    int64_t maxk = 0; for (int w = 0; w < 3; w++) if (hh[w].cap > maxk) maxk = hh[w].cap;
    for (int64_t k = 101; k < maxk; k++) if (HV(0, k) || HV(1, k) || HV(2, k)) fprintf(f, "%lld.0\t0\t%lld\t%lld\t%lld\n", (long long)k, HV(0, k), HV(2, k), HV(1, k));
#undef HV
    fprintf(f, "\n");
    fclose(f); free(ord); free(nm);
    return 0;
}

/* ---------------------------------------------- intervals/intervals.go:88-173 */
static int iv_extend(int32_t *a, const int32_t *b) { if (b[0] > a[1]) return 0; if (b[1] > a[1]) a[1] = b[1]; return 1; }
int64_t orc_flatten(int32_t *se, int64_t len) {
    for (int64_t i = 0, n = len - 1; i < n; i++) {
        if (iv_extend(se + 2 * i, se + 2 * (i + 1))) {
            n++;
            for (int64_t j = i + 1; j < n; j++) {
                if (!iv_extend(se + 2 * i, se + 2 * j)) { i++; se[2 * i] = se[2 * j]; se[2 * i + 1] = se[2 * j + 1]; }
            }
            return i + 1;
        }
    }
    return len;
}
int orc_overlap(const int32_t *se, int64_t n, int32_t start, int32_t end) {
    const int32_t e1 = (int32_t)((uint32_t)end - 1u), s1 = (int32_t)((uint32_t)start - 1u);   /* end-1, start-1 in Go's int32: they wrap */
    for (int64_t left = 0, right = n - 1; left <= right;) {
        int64_t mid = (left + right) / 2;
        int32_t is = se[2 * mid], ie = se[2 * mid + 1];
        if (is > e1) right = mid - 1; else if (ie <= s1) left = mid + 1; else return 1;
    }
    return 0;
}
void orc_intersect(const int32_t *se, int64_t n, int32_t start, int32_t end, int64_t *lo, int64_t *hi) {
    int64_t a = 0, b = n; /* sort.Search: smallest i with End >= start */
    while (a < b) { int64_t m = (a + b) / 2; if (!(se[2 * m + 1] >= start)) a = m + 1; else b = m; }
    *lo = a;
    a = 0; b = n;           /* smallest i with Start > end */
    while (a < b) { int64_t m = (a + b) / 2; if (!(se[2 * m] > end)) a = m + 1; else b = m; }
    *hi = a;
}

/* ---------------------------------------------- filters/utils.go:130-534 (working copy of one alignment) */
#define MAXC 1024
typedef struct {
    int32_t pos, pnext, tlen, refid, nref; uint16_t flag;
    cigop cigar[MAXC]; int nc;
    int s0, slen;                  /* SEQ/QUAL window into the original read */
    const uint8_t *seq, *qual;     /* original read */
    int err;
} waln;
static inline char w_base(const waln *a, int i) { return seq_base(a->seq, a->s0 + i); }
static inline uint8_t w_qual(const waln *a, int i) { return a->qual[a->s0 + i]; }
static int32_t w_end(const waln *a) { int32_t l = 0; for (int i = 0; i < a->nc; i++) l += consumes_ref(a->cigar[i].op) * a->cigar[i].len; return a->pos + l - 1; } /* sam-types.go:769 */
static int32_t read_len_from_cigar(const cigop *c, int nc) { int32_t l = 0; for (int i = 0; i < nc; i++) l += consumes_read(c[i].op) * c[i].len; return l; }
static int is_strict_unmapped(const waln *a) { return (a->flag & 0x4) || a->refid < 0 || a->pos == 0; }        /* utils.go:140 */
static int is_strict_next_unmapped(const waln *a) { return (a->flag & 0x8) || a->nref < 0 || a->pnext == 0; } /* utils.go:144 */

static int soft_start(const waln *a) { /* utils.go:224-234 */
    int32_t s = a->pos;
    for (int i = 0; i < a->nc; i++) { if (a->cigar[i].op == 'S') s -= a->cigar[i].len; else if (a->cigar[i].op != 'H') break; }
    return s;
}
static int soft_end(const waln *a) { /* utils.go:236-248 */
    int32_t end = w_end(a), se = end;
    for (int i = a->nc - 1; i >= 0; i--) { if (a->cigar[i].op == 'S') se += a->cigar[i].len; else if (a->cigar[i].op != 'H') return se; }
    return end;
}
static int read_starts_with_insertion(const cigop *c, int nc, int32_t *len) { /* bqsr.go:287-299 */
    for (int i = 0; i < nc; i++) { if (c[i].op == 'I') { *len = c[i].len; return 1; } if (c[i].op == 'H' || c[i].op == 'S') continue; break; }
    *len = -1; return 0;
}
static int compute_read_coord(const cigop *cv, int nc, int softStart, int refIndex, int *falls) { /* utils.go:267-326 */
    int goal = refIndex - softStart;
    *falls = 0;
    if (goal < 0) return -1;
    int readBases = 0, refBases = 0;
    int fallsInside = 0, endsJustBefore = 0, fallsInsideOrJustBefore = 0;
    int index = 0;
    while (refBases != goal && index < nc) {
        cigop el = cv[index]; index++;
        int elen = el.len, shift = 0;
        if (consumes_ref(el.op) || el.op == 'S') {
            if (refBases + elen < goal) shift = elen; else shift = goal - refBases;
            refBases += shift;
        }
        if (refBases != goal) readBases += consumes_read(el.op) * elen;
        else {
            if (shift >= elen && index == nc) return -1;
            cigop next; next.op = 0; next.len = 0;
            if (shift < elen) fallsInside = (el.op == 'D' || el.op == 'N');
            else {
                next = cv[index]; index++;
                if (next.op == 'I') {
                    readBases += next.len;
                    if (index == nc) return -1;
                    next = cv[index]; index++;
                }
                endsJustBefore = (next.op == 'D' || next.op == 'N');
            }
            fallsInsideOrJustBefore = endsJustBefore || fallsInside;
            if (!fallsInsideOrJustBefore) readBases += consumes_read(el.op) * shift;
            else if (endsJustBefore) readBases += consumes_read(el.op) * (shift - 1);
            else if (fallsInside || (endsJustBefore && (next.op == 'D' || next.op == 'N'))) readBases--;
        }
    }
    if (refBases != goal) return -1;
    *falls = fallsInsideOrJustBefore;
    return readBases;
}
static int get_read_coord(const cigop *cv, int nc, int softStart, int refIndex, int tail_right, int *ok) { /* utils.go:335-349 */
    int falls; int rb = compute_read_coord(cv, nc, softStart, refIndex, &falls);
    if (rb == -1) { *ok = 0; return -1; }
    if (tail_right && falls) rb++;
    if (!tail_right && rb == 0) { int32_t fl; if (read_starts_with_insertion(cv, nc, &fl)) { int32_t m = read_len_from_cigar(cv, nc) - 1; rb = fl < m ? fl : m; } }
    *ok = 1; return rb;
}
static int32_t hard_soft_offset(const cigop *c, int nc) { /* utils.go:351-371 */
    int32_t size = 0; int i = 0;
    for (; i < nc; i++) { if (c[i].op == 'H') size += c[i].len; else break; }
    for (; i < nc; i++) { if (c[i].op == 'S') size += c[i].len; else break; }
    return size;
}
static int clip_align_shift(cigop op, int cigarLength) { /* utils.go:377-386 */
    if (op.op == 'I') return -cigarLength;
    if (op.op == 'D' || op.op == 'N') return op.len;
    return 0;
}
static int clean_hard_clipped(cigop *c, int nc) { /* utils.go:473-504 */
    int total = 0, index = 0;
    for (; index < nc; index++) { char o = c[index].op; if (o == 'H' || o == 'D' || o == 'N') total += c[index].len; else break; }
    if (index > 0) { c[0].op = 'H'; c[0].len = total; memmove(c + 1, c + index, sizeof(cigop) * (nc - index)); nc = 1 + nc - index; }
    total = 0; index = nc - 1;
    for (; index >= 0; index--) { char o = c[index].op; if (o == 'H' || o == 'D' || o == 'N') total += c[index].len; else break; }
    if (index < nc - 1) { c[index + 1].op = 'H'; c[index + 1].len = total; nc = index + 2; }
    return nc;
}
static int hard_clip_cigar(const waln *a, int start, int stop, cigop *out) { /* utils.go:407-471 */
    const cigop *cv = a->cigar; int nc = a->nc;
    int index = 0, total = stop - start + 1, ashift = 0, no = 0;
    if (start == 0) {
        int ci = 0;
        for (int k = 0; k < nc; k++) { ci = k; if (cv[k].op != 'H') break; total += cv[k].len; } /* Go range: ci ends at last index if no break */
        for (; index <= stop && ci < nc; ci++) {
            cigop op = cv[ci]; int L = op.len; int shift = consumes_read(op.op) * L;
            if (index + shift == stop + 1) {
                ashift += clip_align_shift(op, L);
                out[no].op = 'H'; out[no].len = total + ashift; no++;
            } else if (index + shift > stop + 1) {
                int after = L - (stop - index + 1);
                ashift += clip_align_shift(op, stop - index + 1);
                out[no].op = 'H'; out[no].len = total + ashift; no++;
                out[no].op = op.op; out[no].len = after; no++;
            }
            index += shift;
            ashift += clip_align_shift(op, shift);
        }
        for (; ci < nc; ci++) out[no++] = cv[ci];
    } else {
        int ci = 0;
        for (; index < start && ci < nc; ci++) {
            cigop op = cv[ci]; int L = op.len; int shift = consumes_read(op.op) * L;
            if (index + shift < start) out[no++] = op;
            else {
                int after = start - index;
                ashift += clip_align_shift(op, L - (start - index));
                if (op.op == 'H') total += after; else { out[no].op = op.op; out[no].len = after; no++; }
            }
            index += shift;
        }
        for (; ci < nc; ci++) { cigop op = cv[ci]; ashift += clip_align_shift(op, op.len); if (op.op == 'H') total += op.len; }
        out[no].op = 'H'; out[no].len = total + ashift; no++;
    }
    return clean_hard_clipped(out, no);
}
static void hard_clip(waln *a, int start, int stop) { /* utils.go:388-405 */
    if (a->nc + 3 > MAXC) { a->err = -5; return; }
    cigop clipped[MAXC]; int ncl = hard_clip_cigar(a, start, stop, clipped);
    int readLength = a->slen, newLength = readLength - (stop - start + 1);
    int copyStart = 0; if (start == 0) copyStart = stop + 1;
    if (newLength < 0 || copyStart + newLength > readLength) { a->err = -4; a->slen = 0; return; } /* Go: slice bounds panic */
    int32_t shift = hard_soft_offset(clipped, ncl) - hard_soft_offset(a->cigar, a->nc);
    a->s0 += copyStart; a->slen = newLength;
    memcpy(a->cigar, clipped, sizeof(cigop) * ncl); a->nc = ncl;
    if (start == 0 && !is_strict_unmapped(a)) a->pos += shift;
}
static void hard_clip_adaptor(waln *a) { /* utils.go:148-222 */
    int wellDefined = 0, alnEnd = -1;
    if (a->tlen != 0 && (a->flag & 1) && !is_strict_unmapped(a) && !is_strict_next_unmapped(a) && (((a->flag & 0x10) != 0) != ((a->flag & 0x20) != 0))) {
        if (a->flag & 0x10) { alnEnd = w_end(a); wellDefined = alnEnd > a->pnext; }
        else { wellDefined = a->pos <= a->pnext + a->tlen; alnEnd = -1; }
    }
    if (!wellDefined) return;
    int boundary = (a->flag & 0x10) ? (int)a->pnext - 1 : (int)a->pos + abs((int)a->tlen);
    /* isInsideRead :172-180 */
    if (boundary < (int)a->pos) return;
    if (alnEnd < 0) alnEnd = w_end(a);
    if (boundary > alnEnd) return;
    int ok;
    if (a->flag & 0x10) {
        int stop = get_read_coord(a->cigar, a->nc, soft_start(a), boundary, 0, &ok);
        if (!ok) { a->err = -3; return; }
        hard_clip(a, 0, stop);
    } else {
        int start = get_read_coord(a->cigar, a->nc, soft_start(a), boundary, 1, &ok);
        if (!ok) { a->err = -3; return; }
        hard_clip(a, start, a->slen - 1);
    }
}
static void hard_clip_soft_clipped(waln *a) { /* utils.go:506-534 */
    int readIndex = 0, cutLeft = -1, cutRight = -1, rightTail = 0;
    for (int i = 0; i < a->nc; i++) {
        char key = a->cigar[i].op; int ln = a->cigar[i].len;
        if (key == 'S') { if (rightTail) cutRight = readIndex; else cutLeft = readIndex + ln - 1; }
        else if (key != 'H') rightTail = 1;
        readIndex += consumes_read(key) * ln;
    }
    if (cutRight >= 0) hard_clip(a, cutRight, a->slen - 1);
    if (cutLeft >= 0) hard_clip(a, 0, cutLeft);
}

/* ---------------------------------------------- filters/bqsr.go covariates */
static inline int base_index(char b) { switch (b) { case 'A': case 'a': case '*': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': return 3; } return -1; } /* :55-62 */
static inline int base_to_int(uint8_t b) { switch (b) { case 'a': case 'A': case '*': return 1; case 'c': case 'C': return 2; case 'g': case 'G': return 3; case 't': case 'T': return 4; } return 0; } /* :247-252 */
static inline char base_complement(char b) { switch (b) { case 'A': case 'a': return 'T'; case 'C': case 'c': return 'G'; case 'G': case 'g': return 'C'; case 'T': case 't': return 'A'; } return b; } /* :303-310 */

static int32_t key_from_context(const char *dna, int start, int end) { /* :64-76 */
    int32_t key = end - start; unsigned off = 4;
    for (int i = start; i < end; i++) { int bi = base_index(dna[i]); if (bi == -1) return -1; key |= bi << off; off += 2; }
    return key;
}
/* contextWith :87-131 with contextSize = 2. returns count of keys, or -100 where the Go code would panic (index -1) */
static int context_with(const char *bases, int readLength, int32_t *keys) {
    const int contextSize = 2; int32_t mask = (3 | (3 << 2)) << 4; (void)mask;
    mask = 0; for (int i = 0; i < contextSize; i++) mask = (mask << 2) | 3; mask <<= 4; /* createMask :78-83 */
    int nk = 0;
    for (int i = 1; i < contextSize && i <= readLength; i++) keys[nk++] = -1;
    if (readLength < contextSize) return nk;
    unsigned newBaseOffset = 2 * (contextSize - 1) + 4;
    int32_t currentKey = key_from_context(bases, 0, contextSize);
    keys[nk++] = currentKey;
    int currentNPenalty = 0;
    if (currentKey == -1) {
        currentKey = 0; currentNPenalty = contextSize - 1;
        unsigned offset = newBaseOffset;
        for (;;) {
            if (currentNPenalty < 0) return -100; /* Go: index out of range panic */
            if (bases[currentNPenalty] == 'N') break;
            int bi = base_index(bases[currentNPenalty]);
            currentKey |= (int32_t)((uint32_t)bi << offset);
            offset -= 2; currentNPenalty--;
        }
    }
    for (int ci = contextSize; ci < readLength; ci++) {
        int bi = base_index(bases[ci]);
        if (bi == -1) { currentNPenalty = contextSize; currentKey = 0; }
        else { currentKey = (currentKey >> 2) & mask; currentKey |= bi << newBaseOffset; currentKey |= contextSize; }
        if (currentNPenalty == 0) keys[nk++] = currentKey; else { currentNPenalty--; keys[nk++] = -1; }
    }
    return nk;
}
/* computeStrandedClippedSeq :312-362 ; returns 0 for "nil" */
static int stranded_clipped_seq(const waln *a, char *newSeq) {
    int L = a->slen, leftPos = L;
    for (int i = 0; i < leftPos; i++) if (w_qual(a, i) > 2) { leftPos = i; break; }
    int rightPos = leftPos - 1;
    for (int i = L - 1; i >= leftPos; i--) if (w_qual(a, i) > 2) { rightPos = i; break; }
    if (leftPos > rightPos) return 0;
    if (a->flag & 0x10) {
        int j = -1;
        for (int i = rightPos + 1; i < L; i++) newSeq[++j] = 'N';
        for (int i = rightPos; i >= leftPos; i--) newSeq[++j] = base_complement(w_base(a, i));
        for (int i = 0; i < leftPos; i++) newSeq[++j] = 'N';
    } else {
        for (int i = 0; i < leftPos; i++) newSeq[i] = 'N';
        for (int i = leftPos; i <= rightPos; i++) newSeq[i] = w_base(a, i);
        for (int i = rightPos + 1; i < L; i++) newSeq[i] = 'N';
    }
    return 1;
}
/* computeBaseContextCovariate :140-146; returns number of keys (0 if none) or -100 */
static int base_context_covariate(const waln *a, char *scratch, int32_t *keys) {
    int have = stranded_clipped_seq(a, scratch);
    int nk = context_with(scratch, have ? a->slen : 0, keys);
    if (nk < 0) return nk;
    if (a->flag & 0x10) for (int i = 0, j = nk - 1; i < j; i++, j--) { int32_t t = keys[i]; keys[i] = keys[j]; keys[j] = t; }
    return nk;
}
static void prepare_cycle(uint16_t flag, int seqlen, int *cycleFactor, int *increment) { /* :376-383 */
    int reversed = (flag & 0x10) >> 4, last = (flag & 0x80) >> 7;
    int rof = 1 - 2 * last;
    *cycleFactor = rof + reversed * (seqlen - 1) * rof;
    *increment = (1 - 2 * reversed) * rof;
}

/* ---------------------------------------------- bqsr.go:225-244 recalibrateAln */
static int recalibrate_aln(const orc_reads *r, const orc_header *h, int64_t i, const waln *a) {
    if (r->opt_flags && (r->opt_flags[i] & 1)) return 0;   /* _, found := aln.TAGS.Get(sr); if found { return false } (bqsr.go:226-229) */
    if (!(r->mapq[i] > 0 && r->mapq[i] < 255)) return 0;
    if (a->flag & (0x100 | 0x400 | 0x200)) return 0;
    if (is_strict_unmapped(a)) return 0;
    if (!(a->pos > 0)) return 0;
    if (!(r->lseq[i] > 0)) return 0;
    /* SEQ.Len()==len(QUAL): the columnar layout always has one qual byte per base */
    if (r->rg[i] < 0) return 0;
    if (a->refid >= h->n_contigs || !(a->pos <= h->contig_len[a->refid])) return 0; /* alignmentAgreesWithHeader utils.go:130-138 */
    for (int k = 0; k < a->nc; k++) if (a->cigar[k].op == 'N') return 0;
    return r->lseq[i] == read_len_from_cigar(a->cigar, a->nc);
}

static int load_waln(const orc_reads *r, int64_t i, waln *a) {
    a->pos = r->pos[i]; a->pnext = r->pnext[i]; a->tlen = r->tlen[i]; a->refid = r->refid[i]; a->nref = r->nref[i]; a->flag = r->flag[i];
    int nc = (int)(r->cigar_off[i + 1] - r->cigar_off[i]);
    if (nc + 3 > MAXC) return -5;
    for (int k = 0; k < nc; k++) a->cigar[k] = dec(r->cigar[r->cigar_off[i] + k]);
    a->nc = nc; a->s0 = 0; a->slen = r->lseq[i]; a->seq = r->seq + r->seq_off[i]; a->qual = r->qual + r->qual_off[i]; a->err = 0;
    return 0;
}

typedef struct {
    const orc_reads *r; const orc_header *h; const uint8_t *ref; const uint64_t *ref_off; const int32_t *sites; const uint64_t *site_off;
    orc_tables *t; orc_tables *priv; int nt; _Atomic(int) err;
} gather_ctx;
#define TQ(t, cov, q) ((int64_t)(cov) * ORC_NQ + (q))
#define TC(t, cov, q, cyc) ((((int64_t)(cov) * ORC_NQ + (q)) * (2 * (int64_t)(t)->max_cycle + 1)) + (cyc) + (t)->max_cycle)
#define TX(t, cov, q, ctx) ((((int64_t)(cov) * ORC_NQ + (q)) * ORC_NCTX) + (ctx))

static void gather_worker(void *p, int tid, int nt) { /* bqsr.go:471-540 one range of the RangeReduce */
    gather_ctx *c = (gather_ctx *)p; const orc_reads *r = c->r; orc_tables *t = &c->priv[tid];
    int64_t lo = r->n * tid / nt, hi = r->n * (tid + 1) / nt;
    int cap = 0; int *snps = NULL; char *scs = NULL; int32_t *ctxk = NULL; uint8_t *skip = NULL;
    waln *a = (waln *)malloc(sizeof(waln));
    for (int64_t i = lo; i < hi; i++) {
        int le = load_waln(r, i, a);
        if (le) { atomic_store(&c->err, le); continue; }
        if (!recalibrate_aln(r, c->h, i, a)) continue;
        hard_clip_adaptor(a);
        if (a->err) { atomic_store(&c->err, a->err); continue; }
        if (a->slen == 0) continue;
        hard_clip_soft_clipped(a);
        if (a->err) { atomic_store(&c->err, a->err); continue; }
        if (a->slen == 0) continue;
        int L = a->slen;
        if (L > cap) { cap = L + 64; snps = (int *)realloc(snps, sizeof(int) * cap); scs = (char *)realloc(scs, cap); ctxk = (int32_t *)realloc(ctxk, 4 * cap); skip = (uint8_t *)realloc(skip, cap); }
        /* calculateSkipSlice :389-414 */
        memset(skip, 0, L);
        {
            int ss = soft_start(a), se = soft_end(a);
            const int32_t *sv = c->sites + 2 * c->site_off[a->refid]; int64_t ns = (int64_t)(c->site_off[a->refid + 1] - c->site_off[a->refid]);
            int64_t s0, s1; orc_intersect(sv, ns, (int32_t)ss, (int32_t)se, &s0, &s1);
            for (int64_t s = s0; s < s1; s++) {
                int ok; int fs = get_read_coord(a->cigar, a->nc, ss, sv[2 * s], 0, &ok);
                if (!ok || fs < 0) fs = 0;
                int fe = get_read_coord(a->cigar, a->nc, ss, sv[2 * s + 1], 0, &ok);
                if (!ok || fe > L - 1) fe = L - 1;
                for (int k = fs; k <= fe; k++) skip[k] = 1;
            }
        }
        /* computeSnpEvents :254-285 */
        {
            const uint8_t *ref = c->ref + c->ref_off[a->refid]; int64_t reflen = (int64_t)(c->ref_off[a->refid + 1] - c->ref_off[a->refid]);
            for (int k = 0; k < L; k++) snps[k] = 0;
            int ri = 0; int64_t j = a->pos - 1; int bad = 0;
            for (int k = 0; k < a->nc && !bad; k++) {
                int ln = a->cigar[k].len;
                switch (a->cigar[k].op) {
                case 'M': case '=': case 'X':
                    for (int q = 0; q < ln; q++) {
                        if (j >= reflen || ri >= L) { bad = 1; break; } /* Go: index out of range panic */
                        if (base_to_int((uint8_t)w_base(a, ri)) != base_to_int(ref[j])) snps[ri] = 1;
                        ri++; j++;
                    }
                    break;
                case 'D': case 'N': j += ln; break;
                case 'I': case 'S': ri += ln; break;
                }
            }
            if (bad) { atomic_store(&c->err, -6); continue; }
        }
        int cov = c->h->rg_cov[r->rg[i]];
        int cf, inc; prepare_cycle(a->flag, L, &cf, &inc);
        int nk = base_context_covariate(a, scs, ctxk);
        if (nk == -100) { atomic_store(&c->err, -7); continue; }
        for (int k = 0; k < L; k++) {
            if (skip[k]) continue;
            if (base_index(w_base(a, k)) < 0) continue;
            uint8_t qual = w_qual(a, k);
            if (qual < 6) continue;
            int errv = snps[k];
            t->q_obs[TQ(t, cov, qual)]++; t->q_mis[TQ(t, cov, qual)] += errv;
            int cyc = cf + k * inc;
            if (cyc > t->max_cycle || cyc < -t->max_cycle) { atomic_store(&c->err, -8); break; } /* checkCycleCovariate :364-369 */
            t->c_obs[TC(t, cov, qual, cyc)]++; t->c_mis[TC(t, cov, qual, cyc)] += errv;
            if (nk > 0 && ctxk[k] >= 0) { t->x_obs[TX(t, cov, qual, ctxk[k] >> 4)]++; t->x_mis[TX(t, cov, qual, ctxk[k] >> 4)] += errv; }
        }
    }
    free(a); free(snps); free(scs); free(ctxk); free(skip);
}

static size_t tq_n(const orc_tables *t) { return (size_t)t->n_cov * ORC_NQ; }
static size_t tc_n(const orc_tables *t) { return (size_t)t->n_cov * ORC_NQ * (2 * (size_t)t->max_cycle + 1); }
static size_t tx_n(const orc_tables *t) { return (size_t)t->n_cov * ORC_NQ * ORC_NCTX; }

int orc_bqsr_gather(const orc_reads *r, const orc_header *h, const uint8_t *ref, const uint64_t *ref_off,
                    const int32_t *sites, const uint64_t *site_off, orc_tables *t, int nt) {
    if (nt < 1) nt = 1;
    gather_ctx c; memset(&c, 0, sizeof(c)); c.r = r; c.h = h; c.ref = ref; c.ref_off = ref_off; c.sites = sites; c.site_off = site_off; c.t = t; c.nt = nt; atomic_init(&c.err, 0);
    c.priv = (orc_tables *)calloc(nt, sizeof(orc_tables));
    for (int i = 0; i < nt; i++) {
        c.priv[i].n_cov = t->n_cov; c.priv[i].max_cycle = t->max_cycle;
        if (i == 0) { c.priv[0] = *t; continue; }
        c.priv[i].q_obs = (int64_t *)calloc(tq_n(t), 8); c.priv[i].q_mis = (int64_t *)calloc(tq_n(t), 8);
        c.priv[i].c_obs = (int64_t *)calloc(tc_n(t), 8); c.priv[i].c_mis = (int64_t *)calloc(tc_n(t), 8);
        c.priv[i].x_obs = (int64_t *)calloc(tx_n(t), 8); c.priv[i].x_mis = (int64_t *)calloc(tx_n(t), 8);
    }
    parallel_run(nt, gather_worker, &c);
    for (int i = 1; i < nt; i++) { /* bqsrTable.merge :210-223 */
        orc_tables *p = &c.priv[i];
        for (size_t k = 0; k < tq_n(t); k++) { t->q_obs[k] += p->q_obs[k]; t->q_mis[k] += p->q_mis[k]; }
        for (size_t k = 0; k < tc_n(t); k++) { t->c_obs[k] += p->c_obs[k]; t->c_mis[k] += p->c_mis[k]; }
        for (size_t k = 0; k < tx_n(t); k++) { t->x_obs[k] += p->x_obs[k]; t->x_mis[k] += p->x_mis[k]; }
        free(p->q_obs); free(p->q_mis); free(p->c_obs); free(p->c_mis); free(p->x_obs); free(p->x_mis);
    }
    free(c.priv);
    return atomic_load(&c.err);
}

/* ---------------------------------------------- bqsr.go:553-649 */
static const double PRIOR_CACHE[21] = { /* embedded data, bqsr.go:569-591 (= log10(0.9*exp(-d*d/0.5)), last = -MaxFloat64) */
    -0.045757490560675115, -0.9143464543671788, -3.5201133457866898, -7.863058164819208, -13.943180911464733,
    -21.760481585723266, -31.314960187594806, -42.606616717079355, -55.63545117417691, -70.40146355888747,
    -86.90465387121104, -105.14502211114761, -125.1225682786972, -146.83729237385978, -170.2891943966354,
    -195.47827434702398, -222.4045322250256, -251.06796803064023, -281.46858176386786, -313.60637342472336,
    -1.7976931348623157e308};
double orc_prior_cache(int d) { return PRIOR_CACHE[d]; }
static double q2err(double phred) { return gm_pow(10, phred / -10); }       /* :561 */
static double q2prob(double phred) { return 1 - gm_pow(10, phred / -10); }   /* :565 */
static double log10_prior(double emp, double rep) { /* :593-596 */
    int d = (int)(emp - rep); if (d < 0) d = -d; if (d > 20) d = 20; return PRIOR_CACHE[d];
}
static double log10_gamma(int64_t n) { return gm_lgamma((double)n) * 0.4342944819032518 /* math.Log10E */; } /* :598-601 */
static double log10_binom_coef(int64_t n, int64_t k) { return log10_gamma(n + 1) - log10_gamma(k + 1) - log10_gamma(n - k + 1); }
static double log10_binom_prob(int64_t n, int64_t k, double log10p) { /* :607-613 */
    if (log10p == 0.0) return -DBL_MAX;
    double log10MinP = gm_log10(1.0 - gm_pow(10, log10p));
    return log10_binom_coef(n, k) + log10p * (double)k + log10MinP * (double)(n - k);
}
static double log10_likelihood(double emp, int64_t obs, int64_t mis) { /* :615-621 */
    if (obs == 0) return 0.0;
    return log10_binom_prob(obs, mis, emp / -10.0);
}
static uint8_t bayesian_estimate(int64_t obs, int64_t mis, double prior) { /* :623-642 */
    const int64_t maxObs = 2147483647 - 1;
    if (obs > maxObs) { mis = (int64_t)gm_round((double)mis * ((double)maxObs / (double)obs)); obs = maxObs; }
    double max = -DBL_MAX; uint8_t maxI = 0;
    for (int i = 0; i < 61; i++) {
        double fi = (double)i;
        double lp = log10_prior(fi, prior) + log10_likelihood(fi, obs, mis);
        if (max < lp) { max = lp; maxI = (uint8_t)i; }
    }
    return maxI;
}
uint8_t orc_empirical_quality(int64_t obs, int64_t mis, double prior) { /* :644-649 */
    uint8_t e = bayesian_estimate(obs + 1 + 1, mis + 1, prior);
    return e < 93 ? e : 93;
}
void orc_bqsr_finalize(orc_tables *t) { /* :677-694 */
    int64_t nc = 2 * (int64_t)t->max_cycle + 1;
    for (size_t k = 0; k < tq_n(t); k++) if (t->q_obs[k] > 0) t->q_emp[k] = orc_empirical_quality(t->q_obs[k], t->q_mis[k], (double)(k % ORC_NQ));
    for (size_t k = 0; k < tc_n(t); k++) if (t->c_obs[k] > 0) t->c_emp[k] = orc_empirical_quality(t->c_obs[k], t->c_mis[k], (double)((k / nc) % ORC_NQ));
    for (size_t k = 0; k < tx_n(t); k++) if (t->x_obs[k] > 0) t->x_emp[k] = orc_empirical_quality(t->x_obs[k], t->x_mis[k], (double)((k / ORC_NCTX) % ORC_NQ));
}
void orc_combined(const orc_tables *t, int cov, double *rq, int64_t *obs, int64_t *mis, uint8_t *emp, int *exists) { /* :655-674, ascending qual */
    double reported = 0; int64_t o = 0, m = 0; int have = 0;
    for (int q = 0; q < ORC_NQ; q++) {
        int64_t eo = t->q_obs[TQ(t, cov, q)], em = t->q_mis[TQ(t, cov, q)];
        if (eo <= 0) continue;
        if (have) {
            double sumErrors = (double)o * q2err(reported) + (double)eo * q2err((double)q);
            o += eo; m += em;
            reported = -10 * gm_log10(sumErrors / (double)o);
        } else { reported = (double)q; o = eo; m = em; have = 1; }
    }
    *exists = have; *rq = reported; *obs = o; *mis = m;
    *emp = have ? orc_empirical_quality(o, m, reported) : 0;
}
static int err_prob_to_quality(double prob) { /* :701-706 */
    if (prob == 0.0) return 93;
    int q = (int)gm_round(-10 * gm_log10(prob)); if (q > 93) q = 93; if (q < 1) q = 1; return q;
}
void orc_static_quantized(const uint8_t *sqq_in, int n, uint8_t *ss) { /* :710-743 */
    uint8_t quals[256]; if (n > 256) n = 256; memcpy(quals, sqq_in, n);
    memset(ss, 0, 254);
    for (int i = 0; i < 6; i++) ss[i] = (uint8_t)i;
    if (n == 1) { for (int i = 6; i < 254; i++) ss[i] = quals[0]; return; }
    for (int i = 1; i < n; i++) { uint8_t v = quals[i]; int j = i; while (j > 0 && quals[j - 1] > v) { quals[j] = quals[j - 1]; j--; } quals[j] = v; }
    uint8_t prevQual = 6; double prevProb = q2prob((double)prevQual);
    for (int k = 0; k < n; k++) {
        uint8_t nextQual = quals[k];
        for (uint8_t i = prevQual; i < nextQual; i++) {
            double nextProb = q2prob((double)nextQual), iProb = q2prob((double)i);
            if (iProb - prevProb > nextProb - iProb) ss[i] = nextQual; else ss[i] = prevQual;
            prevProb = nextProb; prevQual = nextQual;
        }
    }
    for (int i = prevQual; i < 254; i++) ss[i] = prevQual;
}
typedef struct { int next; double errorRate; int64_t nobs, leafNobs, nerrors; } qinterval; /* :745-751 */
static double calc_error_rate(int64_t nobs, int64_t nerr) { if (nobs == 0) return 0.0; return (double)(nerr + 1) / (double)(nobs + 1); }
static double leaf_penalty(int k, qinterval *iv, double globalErrorRate) { /* :780-786 */
    if (k <= 6) return 0.0;
    return fabs(gm_log10(iv[k].errorRate) - gm_log10(globalErrorRate)) * (double)iv[k].leafNobs;
}
static double merge_penalty(int i, int j, qinterval *iv, int n) { /* :795-818 */
    int64_t mn = iv[i].nobs + iv[j].nobs, me = iv[i].nerrors + iv[j].nerrors;
    double mer = calc_error_rate(mn, me);
    if (mer == 0) return 0.0;
    double sumI = 0, sumJ = 0;
    for (int k = i; k < j; k++) sumI += leaf_penalty(k, iv, mer);
    int kend = iv[j].next >= 0 ? iv[j].next : n;
    for (int k = j; k < kend; k++) sumJ += leaf_penalty(k, iv, mer);
    return sumI + sumJ;
}
static int merge_minimal(qinterval *iv, int n) { /* :820-850 */
    int i = 0, j = iv[0].next; if (j < 0) return 0;
    int minI = i; double mp = merge_penalty(i, j, iv, n);
    for (;;) {
        i = j; j = iv[i].next; if (j < 0) break;
        double p = merge_penalty(i, j, iv, n);
        if (p < mp) { minI = i; mp = p; }
    }
    qinterval *a = &iv[minI], *b = &iv[a->next];
    int64_t mn = a->nobs + b->nobs, me = a->nerrors + b->nerrors;
    a->next = b->next; a->nobs = mn; a->nerrors = me;
    return 1;
}
void orc_quantized(const orc_tables *t, int levels, int64_t *qmap, uint8_t *scores) { /* :863-899 */
    const int N = 94;
    for (int i = 0; i < N; i++) { qmap[i] = 0; scores[i] = 0; }
    if (levels == 0) { for (int i = 0; i < N; i++) scores[i] = (uint8_t)i; return; }
    for (size_t k = 0; k < tq_n(t); k++) if (t->q_obs[k] > 0) qmap[t->q_emp[k]] += t->q_obs[k];
    qinterval iv[94];
    for (int i = 0; i < N; i++) { /* :760-778 */
        double er = q2err((double)i);
        iv[i].next = (i + 1 == N) ? -1 : i + 1; iv[i].errorRate = er; iv[i].nobs = qmap[i]; iv[i].leafNobs = qmap[i]; iv[i].nerrors = (int64_t)((double)qmap[i] * er);
    }
    for (int n = N; n > levels;) { if (merge_minimal(iv, N)) n--; else break; }
    for (int i = 0; i >= 0;) {
        uint8_t qs;
        int leaf = iv[i].next < 0 ? (i == 93) : (iv[i].next == i + 1); /* :753-758 */
        if (leaf) qs = (uint8_t)i; else qs = (uint8_t)err_prob_to_quality(calc_error_rate(iv[i].nobs, iv[i].nerrors));
        int kend = iv[i].next >= 0 ? iv[i].next : N;
        for (int k = i; k < kend; k++) scores[k] = qs;
        i = iv[i].next;
    }
}

/* ---------------------------------------------- bqsr.go:901-1006 apply */
typedef struct {
    const orc_reads *r; const orc_header *h; const orc_tables *t; const uint8_t *quant; const uint8_t *stat; int have_stat;
    double *rq; int64_t *cobs, *cmis; int *cexists; uint16_t *memo; _Atomic(int) err;
} apply_ctx;
static double hierarchical_estimate(const apply_ctx *c, int cov, int q, int cyc, int ctx) { /* :901-919 */
    const orc_tables *t = c->t; double epsilon = c->rq[cov];
    double dG = 0, dQ = 0;
    dG = (double)orc_empirical_quality(c->cobs[cov], c->cmis[cov], epsilon) - epsilon; /* empiricalReadGroupEntry != nil here */
    if (t->q_obs[TQ(t, cov, q)] > 0) dQ = (double)orc_empirical_quality(t->q_obs[TQ(t, cov, q)], t->q_mis[TQ(t, cov, q)], dG + epsilon) - dG - epsilon;
    double dC = 0; double cp = dQ + dG + epsilon;
    if (t->c_obs[TC(t, cov, q, cyc)] > 0) dC = (double)orc_empirical_quality(t->c_obs[TC(t, cov, q, cyc)], t->c_mis[TC(t, cov, q, cyc)], cp) - cp;
    if (ctx >= 0 && t->x_obs[TX(t, cov, q, ctx >> 4)] > 0) dC += (double)orc_empirical_quality(t->x_obs[TX(t, cov, q, ctx >> 4)], t->x_mis[TX(t, cov, q, ctx >> 4)], cp) - cp;
    return cp + dC;
}
static void apply_worker(void *p, int tid, int nt) {
    apply_ctx *c = (apply_ctx *)p; const orc_reads *r = c->r; const orc_tables *t = c->t;
    int64_t lo = r->n * tid / nt, hi = r->n * (tid + 1) / nt;
    int cap = 0; char *scs = NULL; int32_t *ctxk = NULL; waln *a = (waln *)malloc(sizeof(waln));
    int64_t ncyc = 2 * (int64_t)t->max_cycle + 1;
    for (int64_t i = lo; i < hi; i++) {
        if (r->rg[i] < 0) { atomic_store(&c->err, -9); continue; } /* readGroupCovariate panics :38 */
        int cov = c->h->rg_cov[r->rg[i]];
        if (!c->cexists[cov]) continue; /* :950-953 */
        a->flag = r->flag[i]; a->s0 = 0; a->slen = r->lseq[i]; a->seq = r->seq + r->seq_off[i]; a->qual = r->qual + r->qual_off[i];
        int L = a->slen;
        if (L > cap) { cap = L + 64; scs = (char *)realloc(scs, cap); ctxk = (int32_t *)realloc(ctxk, 4 * cap); }
        int cf, inc; prepare_cycle(a->flag, L, &cf, &inc);
        int nk = base_context_covariate(a, scs, ctxk);
        if (nk == -100) { atomic_store(&c->err, -7); continue; }
        uint8_t *qual = r->qual + r->qual_off[i];
        for (int k = 0; k < L; k++) {
            uint8_t q = qual[k];
            if (q < 6) continue;
            int cyc = cf + k * inc;
            if (cyc > t->max_cycle || cyc < -t->max_cycle) { atomic_store(&c->err, -8); break; }
            int ctx = ctxk[k];
            size_t mi = ((((size_t)cov * ORC_NQ + q) * ncyc) + (size_t)(cyc + t->max_cycle)) * 17 + (size_t)(ctx >= 0 ? (ctx >> 4) : 16);
            uint16_t mv = __atomic_load_n(&c->memo[mi], __ATOMIC_RELAXED);
            if (!mv) {
                double est = hierarchical_estimate(c, cov, q, cyc, ctx);
                int ri = (int)gm_round(est); if (ri > 93) ri = 93; if (ri < 1) ri = 1;
                uint8_t nq = c->quant[ri];
                if (c->have_stat) nq = c->stat[nq];
                mv = (uint16_t)(0x100 | nq);
                __atomic_store_n(&c->memo[mi], mv, __ATOMIC_RELAXED);
            }
            qual[k] = (uint8_t)(mv & 0xff);
        }
    }
    free(a); free(scs); free(ctxk);
}
int orc_bqsr_apply(const orc_reads *r, const orc_header *h, const orc_tables *t, int quantize_levels, const uint8_t *sqq, int n_sqq, int nt) {
    if (nt < 1) nt = 1;
    apply_ctx c; memset(&c, 0, sizeof(c)); c.r = r; c.h = h; c.t = t; atomic_init(&c.err, 0);
    int64_t qmap[94]; uint8_t quant[94]; uint8_t stat[254];
    orc_quantized(t, quantize_levels, qmap, quant); c.quant = quant;
    if (n_sqq > 0) { orc_static_quantized(sqq, n_sqq, stat); c.stat = stat; c.have_stat = 1; }
    c.rq = (double *)calloc(t->n_cov, 8); c.cobs = (int64_t *)calloc(t->n_cov, 8); c.cmis = (int64_t *)calloc(t->n_cov, 8); c.cexists = (int *)calloc(t->n_cov, sizeof(int));
    for (int cov = 0; cov < t->n_cov; cov++) { uint8_t e; orc_combined(t, cov, &c.rq[cov], &c.cobs[cov], &c.cmis[cov], &e, &c.cexists[cov]); }
    size_t memo_n = (size_t)t->n_cov * ORC_NQ * (2 * (size_t)t->max_cycle + 1) * 17;
    c.memo = (uint16_t *)calloc(memo_n, 2);
    parallel_run(nt, apply_worker, &c);
    free(c.rq); free(c.cobs); free(c.cmis); free(c.cexists); free(c.memo);
    return atomic_load(&c.err);
}

/* ---------------------------------------------- print-bqsr.go:49-298 */
static int ilen(int64_t v) { char b[32]; return snprintf(b, sizeof b, "%lld", (long long)v); }
static int imax(int a, int b) { return a > b ? a : b; }
static void key_to_string(int32_t key, char *out) { /* bqsr.go:166-178 */
    int length = key & 0xF; int32_t rk = key >> 4; int n = 0;
    for (int i = 0; i < length; i++) { out[n++] = "ACGT"[rk & 3]; rk >>= 2; }
    out[n] = 0;
}
typedef struct { int cov; int q; int is_cycle; char text[16]; int64_t obs, mis; uint8_t emp; const char *rgname; } rt2row;
static int rt2cmp(const void *a, const void *b) {
    const rt2row *x = (const rt2row *)a, *y = (const rt2row *)b;
    int c = strcmp(x->rgname, y->rgname); if (c) return c;
    if (x->q != y->q) return x->q < y->q ? -1 : 1;
    return strcmp(x->text, y->text);
}
static int strpcmp(const void *a, const void *b) { return strcmp(*(const char *const *)a, *(const char *const *)b); }
int orc_bqsr_report(const orc_tables *t, const char *const *cov_names, const char *prefix, const char *path) {
    FILE *f = fopen(path, "w"); if (!f) return -1;
    fprintf(f, "#:%sReport.v1.1:5\n", prefix);
    fprintf(f, "#:%sTable:2:17:%%s:%%s:;\n", prefix);
    fprintf(f, "#:%sTable:Arguments:Recalibration argument collection values used in this run\n", prefix);
    static const char *args[] = {
        "Argument                    Value                                                                   ",
        "binary_tag_name             null                                                                    ",
        "covariate                   ReadGroupCovariate,QualityScoreCovariate,ContextCovariate,CycleCovariate",
        "default_platform            null                                                                    ",
        "deletions_default_quality   45                                                                      ",
        "force_platform              null                                                                    ",
        "indels_context_size         3                                                                       ",
        "insertions_default_quality  45                                                                      ",
        "low_quality_tail            2                                                                       ",
        "maximum_cycle_value         500                                                                     ",
        "mismatches_context_size     2                                                                       ",
        "mismatches_default_quality  -1                                                                      ",
        "no_standard_covs            false                                                                   ",
        "quantizing_levels           16                                                                      ",
        "recalibration_report        null                                                                    ",
        "run_without_dbsnp           false                                                                   ",
        "solid_nocall_strategy       THROW_EXCEPTION                                                         ",
        "solid_recal_mode            SET_Q_ZERO                                                              "};
    for (size_t i = 0; i < sizeof(args) / sizeof(args[0]); i++) fprintf(f, "%s\n", args[i]);
    fprintf(f, "\n");
    /* quantization table :49-76 */
    {
        int64_t obs[94]; uint8_t sc[94]; orc_quantized(t, 16, obs, sc);
        fprintf(f, "#:%sTable:3:%d:%%d:%%d:%%d:;\n", prefix, 94);
        fprintf(f, "#:%sTable:Quantized:Quality quantization map\n", prefix);
        int w1 = 12, w2 = 5, w3 = 14;
        for (int i = 0; i < 94; i++) { w1 = imax(w1, ilen(i)); w2 = imax(w2, ilen(obs[i])); w3 = imax(w3, ilen(sc[i])); }
        fprintf(f, "%-*s  %-*s  %-*s\n", w1, "QualityScore", w2, "Count", w3, "QuantizedScore");
        for (int i = 0; i < 94; i++) fprintf(f, "%*d  %*lld  %*d\n", w1, i, w2, (long long)obs[i], w3, (int)sc[i]);
        fprintf(f, "\n");
    }
    /* RecalTable0 :78-122 */
    {
        int nrg = 0; const char **names = (const char **)malloc(sizeof(char *) * (t->n_cov + 1));
        double *rq = (double *)calloc(t->n_cov, 8); int64_t *o = (int64_t *)calloc(t->n_cov, 8), *m = (int64_t *)calloc(t->n_cov, 8); uint8_t *e = (uint8_t *)calloc(t->n_cov, 1);
        int wrg = 9, wev = 9, wemp = 16, wrep = 18, wobs = 12, werr = 6;
        for (int c = 0; c < t->n_cov; c++) {
            int ex; orc_combined(t, c, &rq[c], &o[c], &m[c], &e[c], &ex); if (!ex) continue;
            names[nrg++] = cov_names[c];
            char b[64]; wrg = imax(wrg, (int)strlen(cov_names[c])); wemp = imax(wemp, ilen(e[c]) + 5);
            wrep = imax(wrep, snprintf(b, sizeof b, "%.4f", rq[c])); wobs = imax(wobs, ilen(o[c])); werr = imax(werr, ilen(m[c]) + 3);
        }
        fprintf(f, "#:%sTable:6:%d:%%s:%%s:%%.4f:%%.4f:%%d:%%.2f:;\n", prefix, nrg);
        fprintf(f, "#:%sTable:RecalTable0:\n", prefix);
        fprintf(f, "%-*s  %-*s  %-*s  %-*s  %-*s  %-*s\n", wrg, "ReadGroup", wev, "EventType", wemp, "EmpiricalQuality", wrep, "EstimatedQReported", wobs, "Observations", werr, "Errors");
        qsort(names, nrg, sizeof(char *), strpcmp);
        for (int k = 0; k < nrg; k++) {
            int c = 0; for (; c < t->n_cov; c++) if (cov_names[c] == names[k]) break;
            fprintf(f, "%-*s  %-*s  %*d.0000  %*.4f  %*lld  %*lld.00\n", wrg, names[k], wev, "M", wemp - 5, (int)e[c], wrep, rq[c], wobs, (long long)o[c], werr - 3, (long long)m[c]);
        }
        fprintf(f, "\n");
        free(names); free(rq); free(o); free(m); free(e);
    }
    /* RecalTable1 :124-175 */
    {
        int n = 0; rt2row *rows = (rt2row *)malloc(sizeof(rt2row) * (tq_n(t) + 1));
        int wrg = 9, wq = 12, wev = 9, wemp = 16, wobs = 12, werr = 6;
        for (int c = 0; c < t->n_cov; c++) for (int q = 0; q < ORC_NQ; q++) {
            size_t k = TQ(t, c, q); if (t->q_obs[k] <= 0) continue;
            rt2row *r = &rows[n++]; r->cov = c; r->q = q; r->text[0] = 0; r->obs = t->q_obs[k]; r->mis = t->q_mis[k]; r->emp = t->q_emp[k]; r->rgname = cov_names[c];
            wrg = imax(wrg, (int)strlen(cov_names[c])); wq = imax(wq, ilen(q)); wemp = imax(wemp, ilen(r->emp) + 5); wobs = imax(wobs, ilen(r->obs)); werr = imax(werr, ilen(r->mis) + 3);
        }
        fprintf(f, "#:%sTable:6:%d:%%s:%%d:%%s:%%.4f:%%d:%%.2f:;\n", prefix, n);
        fprintf(f, "#:%sTable:RecalTable1:\n", prefix);
        fprintf(f, "%-*s  %-*s  %-*s  %-*s  %-*s  %-*s\n", wrg, "ReadGroup", wq, "QualityScore", wev, "EventType", wemp, "EmpiricalQuality", wobs, "Observations", werr, "Errors");
        qsort(rows, n, sizeof(rt2row), rt2cmp);
        for (int k = 0; k < n; k++) fprintf(f, "%-*s  %*d  %-*s  %*d.0000  %*lld  %*lld.00\n", wrg, rows[k].rgname, wq, rows[k].q, wev, "M", wemp - 5, (int)rows[k].emp, wobs, (long long)rows[k].obs, werr - 3, (long long)rows[k].mis);
        fprintf(f, "\n");
        free(rows);
    }
    /* RecalTable2 :183-266 */
    {
        int64_t ncyc = 2 * (int64_t)t->max_cycle + 1; size_t n = 0, cap = 1024; rt2row *rows = (rt2row *)malloc(sizeof(rt2row) * cap);
        int wrg = 9, wq = 12, wcv = 14, wcn = 13, wev = 9, wemp = 16, wobs = 12, werr = 6;
        for (int c = 0; c < t->n_cov; c++) for (int q = 0; q < ORC_NQ; q++) {
            for (int64_t cy = -t->max_cycle; cy <= t->max_cycle; cy++) {
                size_t k = TC(t, c, q, cy); if (t->c_obs[k] <= 0) continue;
                if (n == cap) { cap *= 2; rows = (rt2row *)realloc(rows, sizeof(rt2row) * cap); }
                rt2row *r = &rows[n++]; r->cov = c; r->q = q; r->is_cycle = 1; snprintf(r->text, sizeof r->text, "%lld", (long long)cy); r->obs = t->c_obs[k]; r->mis = t->c_mis[k]; r->emp = t->c_emp[k]; r->rgname = cov_names[c];
            }
            for (int x = 0; x < ORC_NCTX; x++) {
                size_t k = TX(t, c, q, x); if (t->x_obs[k] <= 0) continue;
                if (n == cap) { cap *= 2; rows = (rt2row *)realloc(rows, sizeof(rt2row) * cap); }
                rt2row *r = &rows[n++]; r->cov = c; r->q = q; r->is_cycle = 0; key_to_string((x << 4) | 2, r->text); r->obs = t->x_obs[k]; r->mis = t->x_mis[k]; r->emp = t->x_emp[k]; r->rgname = cov_names[c];
            }
        }
        (void)ncyc;
        for (size_t k = 0; k < n; k++) { rt2row *r = &rows[k]; wrg = imax(wrg, (int)strlen(r->rgname)); wq = imax(wq, ilen(r->q)); wcv = imax(wcv, (int)strlen(r->text)); wemp = imax(wemp, ilen(r->emp) + 5); wobs = imax(wobs, ilen(r->obs)); werr = imax(werr, ilen(r->mis) + 3); }
        fprintf(f, "#:%sTable:8:%zu:%%s:%%d:%%s:%%s:%%s:%%.4f:%%d:%%.2f:;\n", prefix, n);
        fprintf(f, "#:%sTable:RecalTable2:\n", prefix);
        fprintf(f, "%-*s  %-*s  %-*s  %-*s  %-*s  %-*s  %-*s  %-*s\n", wrg, "ReadGroup", wq, "QualityScore", wcv, "CovariateValue", wcn, "CovariateName", wev, "EventType", wemp, "EmpiricalQuality", wobs, "Observations", werr, "Errors");
        qsort(rows, n, sizeof(rt2row), rt2cmp);
        for (size_t k = 0; k < n; k++) fprintf(f, "%-*s  %*d  %-*s  %-*s  %-*s  %*d.0000  %*lld  %*lld.00\n", wrg, rows[k].rgname, wq, rows[k].q, wcv, rows[k].text, wcn, rows[k].is_cycle ? "Cycle" : "Context", wev, "M", wemp - 5, (int)rows[k].emp, wobs, (long long)rows[k].obs, werr - 3, (long long)rows[k].mis);
        fprintf(f, "\n");
        free(rows);
    }
    fclose(f);
    return 0;
}

/* ---------------------------------------------- probes for known-answer tests */
int orc_probe_clip(int32_t pos, uint16_t flag, int32_t pnext, int32_t tlen, int32_t refid, int32_t nref,
                   const uint32_t *cigar, int32_t ncigar, int32_t lseq, int32_t *lo, int32_t *hi, int32_t *newpos, uint32_t *newcigar, int cap) {
    waln *a = (waln *)calloc(1, sizeof(waln));
    a->pos = pos; a->flag = flag; a->pnext = pnext; a->tlen = tlen; a->refid = refid; a->nref = nref;
    for (int k = 0; k < ncigar; k++) a->cigar[k] = dec(cigar[k]);
    a->nc = ncigar; a->s0 = 0; a->slen = lseq;
    hard_clip_adaptor(a);
    if (a->err || a->slen == 0) { int e = a->err ? a->err : -1; free(a); return e; }
    hard_clip_soft_clipped(a);
    if (a->err || a->slen == 0) { int e = a->err ? a->err : -1; free(a); return e; }
    *lo = a->s0; *hi = a->s0 + a->slen; *newpos = a->pos;
    int nc = a->nc; for (int k = 0; k < nc && k < cap; k++) newcigar[k] = enc(a->cigar[k]);
    free(a); return nc;
}
int orc_probe_readcoord(const uint32_t *cigar, int32_t ncigar, int softStart, int refIndex, int tail_right, int *ok) {
    cigop cv[MAXC]; for (int k = 0; k < ncigar; k++) cv[k] = dec(cigar[k]);
    return get_read_coord(cv, ncigar, softStart, refIndex, tail_right, ok);
}
int orc_probe_context(const uint8_t *seq_nibbles, const uint8_t *qual, int32_t lseq, int reversed, int32_t *keys) {
    waln *a = (waln *)calloc(1, sizeof(waln)); a->flag = reversed ? 0x10 : 0; a->s0 = 0; a->slen = lseq; a->seq = seq_nibbles; a->qual = qual;
    char *scs = (char *)malloc(lseq + 1);
    int nk = base_context_covariate(a, scs, keys);
    free(scs); free(a); return nk;
}
void orc_probe_cycle(uint16_t flag, int32_t lseq, int32_t *cycles) { int cf, inc; prepare_cycle(flag, lseq, &cf, &inc); for (int i = 0; i < lseq; i++) cycles[i] = cf + i * inc; }
