/* kaiju_oracle.c -- CPU restatement of Kaiju's per-read classification path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under kaiju_b200/ may include, link or call this file; only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg use it, and only as the checker.
 *
 * Parity status: PINNED.  The reference ships no golden vectors for this path (SURVEY.md section 4),
 * so the oracle is pinned against the reference itself: tests/test_oracle_vs_ref.py runs
 * oracle/_ref/kaiju (the unmodified reference built by oracle/Makefile) and oracle/_ref/libkaijuref.so
 * (FMindex, get_suffix, SeqBufferSeg, lnfact) on seeded inputs and requires identical results, and
 * tests/golden/ holds reference outputs produced by tests/golden/make_golden.py.
 *
 * Every function cites the reference file:line (relative to src/) whose behaviour it restates.  The
 * code is written from the behavioural spec in SURVEY.md section 8a / Appendix A: arrays instead of the
 * reference's linked lists and STL containers, a plain checkpointed rank table instead of the
 * byte-recoded BWT scan.
 */
#include "kaiju_oracle.h"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <limits.h>

#define KO_OCC_SHIFT 7                      /* our own checkpoint spacing: 128 letters */
#define KO_OCC_SIZE (1 << KO_OCC_SHIFT)

struct ko_index {
    /* BWT header (bwt/bwt.c:51-61) */
    int64_t len; int nseq; int alen; char alphabet[64];
    /* suffix-array header + body (bwt/suffixArray.c:282-321) */
    int64_t sa_len, ncheck; int chpt_exp, nbytes, sbits, pbits; int64_t mask, check;
    char **ids; uint64_t *seq_taxon; uint8_t *sa;
    /* FM index (bwt/fmicommon.h:190-217, bwt/compactfmi.c:165-171) */
    int64_t bwtlen; int N1, N2; uint8_t *bwt; int64_t *index1; uint16_t *index2; int32_t startLcode[64];
    uint8_t lcode[256], ncode[256];
    /* derived */
    uint8_t *letters; int64_t C[64]; int64_t *occ; int64_t nocc;
    int64_t quirk_lo, quirk_d[64];   /* checkpoint quirk of indexes with bwtlen = m * 65536, m >= 2 (see rank_) */
    uint8_t trans[256];
};

/* ------------------------------------------------------------------------------------------
 * .fmi loader.  Layout written by mkfmi.c:68-77: BWT header, SA header + body, FMI.
 * ------------------------------------------------------------------------------------------ */
static int rd(void *p, size_t sz, size_t n, FILE *fp) { return fread(p, sz, n, fp) == n ? 0 : -1; }

ko_index *ko_index_load(const char *path) {
    FILE *fp = fopen(path, "rb"); if (!fp) return NULL;
    ko_index *x = (ko_index *)calloc(1, sizeof(ko_index));
    int32_t i32; int bad = 0;
    bad |= rd(&x->len, 8, 1, fp); bad |= rd(&i32, 4, 1, fp); x->nseq = i32; bad |= rd(&i32, 4, 1, fp); x->alen = i32;
    if (bad || x->alen <= 0 || x->alen > 60) { fclose(fp); free(x); return NULL; }
    bad |= rd(x->alphabet, 1, (size_t)x->alen, fp);
    bad |= rd(&x->sa_len, 8, 1, fp); bad |= rd(&x->ncheck, 8, 1, fp);
    bad |= rd(&i32, 4, 1, fp); x->chpt_exp = i32; bad |= rd(&i32, 4, 1, fp); x->nbytes = i32;
    bad |= rd(&i32, 4, 1, fp); x->sbits = i32; bad |= rd(&i32, 4, 1, fp); x->pbits = i32;
    bad |= rd(&x->mask, 8, 1, fp); bad |= rd(&x->check, 8, 1, fp);
    int32_t nseq2 = 0; bad |= rd(&nseq2, 4, 1, fp);
    if (bad) { fclose(fp); free(x); return NULL; }
    x->ids = (char **)calloc((size_t)nseq2, sizeof(char *));
    x->seq_taxon = (uint64_t *)calloc((size_t)nseq2, sizeof(uint64_t));
    for (int i = 0; i < nseq2; i++) {
        uint8_t l = 0; bad |= rd(&l, 1, 1, fp);
        x->ids[i] = (char *)malloc((size_t)l + 1); bad |= l ? rd(x->ids[i], 1, l, fp) : 0; x->ids[i][l] = 0;
        /* ConsumerThread.cpp:812-832: number after the LAST '_' , else the whole name */
        const char *u = strrchr(x->ids[i], '_');
        x->seq_taxon[i] = strtoul(u ? u + 1 : x->ids[i], NULL, 10);
    }
    fseek(fp, (long)nseq2 * 4, SEEK_CUR);            /* seqTermOrder */
    fseek(fp, (long)nseq2 * 8, SEEK_CUR);            /* seqlengths */
    x->sa = (uint8_t *)malloc((size_t)(x->ncheck * x->nbytes) + 8);
    bad |= rd(x->sa, 1, (size_t)(x->ncheck * x->nbytes), fp);
    int32_t alen2 = 0; bad |= rd(&alen2, 4, 1, fp); bad |= rd(&x->bwtlen, 8, 1, fp);
    bad |= rd(&i32, 4, 1, fp); x->N1 = i32; bad |= rd(&i32, 4, 1, fp); x->N2 = i32;
    if (bad || alen2 != x->alen) { fclose(fp); return NULL; }
    x->bwt = (uint8_t *)malloc((size_t)x->bwtlen + 1);
    bad |= rd(x->bwt, 1, (size_t)x->bwtlen, fp);
    x->index1 = (int64_t *)malloc(sizeof(int64_t) * (size_t)x->N1 * x->alen);
    bad |= rd(x->index1, 8, (size_t)x->N1 * x->alen, fp);
    x->index2 = (uint16_t *)malloc(sizeof(uint16_t) * (size_t)x->N2 * x->alen);
    bad |= rd(x->index2, 2, (size_t)x->N2 * x->alen, fp);
    bad |= rd(x->startLcode, 4, (size_t)x->alen + 1, fp);
    fclose(fp);
    if (bad) return NULL;
    /* byte code -> (letter, count) tables, compactfmi.c:75-89 */
    for (int a = 0; a < x->alen; a++) {
        int n = 0, k;
        for (k = x->startLcode[a]; k < x->startLcode[a + 1] - 1; k++) { x->lcode[k] = (uint8_t)a; x->ncode[k] = (uint8_t)n++; }
        x->lcode[k] = (uint8_t)a; x->ncode[k] = 255;
    }
    /* C[] = last index1 row (bwt.c:146-152 reads index1[N1-1][c]) */
    for (int a = 0; a < x->alen; a++) x->C[a] = x->index1[(size_t)(x->N1 - 1) * x->alen + a];
    /* our own rank table over the decoded letters */
    x->letters = (uint8_t *)malloc((size_t)x->bwtlen + 1);
    x->nocc = (x->bwtlen >> KO_OCC_SHIFT) + 1;
    x->occ = (int64_t *)malloc(sizeof(int64_t) * (size_t)x->nocc * x->alen);
    int64_t run[64]; memset(run, 0, sizeof(run));
    for (int64_t k = 0; k < x->bwtlen; k++) {
        if ((k & (KO_OCC_SIZE - 1)) == 0) memcpy(x->occ + (k >> KO_OCC_SHIFT) * x->alen, run, sizeof(int64_t) * x->alen);
        uint8_t c = x->lcode[x->bwt[k]]; x->letters[k] = c; run[c]++;
    }
    if ((x->bwtlen & (KO_OCC_SIZE - 1)) == 0) memcpy(x->occ + (x->bwtlen >> KO_OCC_SHIFT) * x->alen, run, sizeof(int64_t) * x->alen);
    /* Checkpoint quirk of the reference (fmicommon.h:60-73, 88-89, 114-158): when bwtlen is a multiple of 2^16 the first-level
     * checkpoint that positions k >= bwtlen - 128 resolve to (chpt1 = bwtlen >> 16) is the row that holds the letter starts C[]
     * (index1[N1-1]), not a count row, and the last index2 row is relative to the previous first-level checkpoint: FMindex then
     * returns C[c] + #c in the last 2^16 rows before k, i.e. the true value minus #c in BWT[0, bwtlen - 2^16).  Verified against the
     * reference binary (tests/test_oracle_vs_ref.py::test_bwtlen_multiple_of_65536); no effect for bwtlen = 2^16. */
    x->quirk_lo = INT64_MAX; memset(x->quirk_d, 0, sizeof x->quirk_d);
    if ((x->bwtlen & 65535) == 0 && x->bwtlen >= 131072) {
        x->quirk_lo = x->bwtlen - 128;
        const int64_t b = (x->bwtlen - 65536) >> KO_OCC_SHIFT;
        for (int a = 0; a < x->alen; a++) x->quirk_d[a] = x->occ[b * x->alen + a];
    }
    /* alphabet translation, sequence.c:68-97,125-134: unknown letters -> last index */
    memset(x->trans, (uint8_t)(x->alen - 1), 256);
    for (int a = 0; a < x->alen; a++) x->trans[(uint8_t)x->alphabet[a]] = (uint8_t)a;
    return x;
}

void ko_index_free(ko_index *x) {
    if (!x) return;
    for (int i = 0; i < x->nseq; i++) free(x->ids[i]);
    free(x->ids); free(x->seq_taxon); free(x->sa); free(x->bwt); free(x->index1); free(x->index2);
    free(x->letters); free(x->occ); free(x);
}
int64_t ko_index_bwtlen(const ko_index *x) { return x->bwtlen; }
int ko_index_alen(const ko_index *x) { return x->alen; }
int ko_index_nseq(const ko_index *x) { return x->nseq; }
uint64_t ko_index_seq_taxon(const ko_index *x, int i) { return x->seq_taxon[i]; }

/* ------------------------------------------------------------------------------------------
 * FMindex (compactfmi.c:267-307): value = C[ct] + #{p < k : L[p] == ct}.
 * Also accounts the bytes the REFERENCE's scan would have examined (compactfmi.c:201-214,249-256),
 * which is the roofline numerator of SURVEY.md 8d.
 * ------------------------------------------------------------------------------------------ */
static inline int64_t rank_(const ko_index *x, int c, int64_t k) {
    int64_t b = k >> KO_OCC_SHIFT, r = x->C[c] + x->occ[b * x->alen + c];
    const uint8_t *L = x->letters; for (int64_t p = b << KO_OCC_SHIFT; p < k; p++) r += (L[p] == c);
    if (k >= x->quirk_lo) r -= x->quirk_d[c];                      /* the reference's checkpoint quirk, see ko_index_load */
    return r;
}
int64_t ko_fmindex(const ko_index *x, int c, int64_t k) { return rank_(x, c, k); }

static uint64_t ref_scan_bytes(const ko_index *x, int ct, int64_t k) {
    uint64_t n = 0; int64_t p = k; int found = 1;
    int dir = (k & 128) ? 1 : -1;                                  /* fmicommon.h:48-52 */
    int c = 255; if (k < x->bwtlen) { c = x->lcode[x->bwt[k]]; n++; }
    if (c != ct) {
        int64_t stop = k & ~(int64_t)255;
        if (p == stop) found = 0;
        else {
            if (dir > 0) { stop += 256; if (stop >= x->bwtlen) { stop = x->bwtlen; if (k >= x->bwtlen) p = stop - 1; } stop -= 1; }
            if (p == stop) found = 0;
            else { p += dir; n++; while (x->lcode[x->bwt[p]] != ct) { if (p == stop) { found = 0; break; } p += dir; n++; } }
        }
    }
    if (found) {                                                   /* fmi_bwt2number hops on saturated codes */
        while (x->ncode[x->bwt[p]] == 255) {
            int64_t lim = dir > 0 ? x->bwtlen - 1 : 0;
            if (p == lim) break;
            p += dir; n++;
            while (x->lcode[x->bwt[p]] != ct) { if (p == lim) break; p += dir; n++; }
            if (x->lcode[x->bwt[p]] != ct) break;
        }
    }
    return n;
}
static inline int64_t fmindex_counted(const ko_index *x, int c, int64_t k, ko_counters *ctr) {
    if (ctr) { ctr->fmindex++; ctr->scanned_bytes += ref_scan_bytes(x, c, k); }
    return rank_(x, c, k);
}

/* InitialSI (bwt.c:146-152) */
static void initial_si(const ko_index *x, int c, int64_t si[2], ko_counters *ctr) {
    if (ctr) ctr->initial_si++;
    si[0] = x->C[c]; si[1] = (c < x->alen - 1) ? x->C[c + 1] : x->bwtlen;
}
/* UpdateSI (bwt.c:160-173): in place on success, untouched on failure */
static int update_si(const ko_index *x, int c, int64_t si[2], int64_t out[2], ko_counters *ctr) {
    if (ctr) ctr->update_si++;
    int64_t a = fmindex_counted(x, c, si[0], ctr), b = fmindex_counted(x, c, si[1], ctr);
    if (a >= b) return 0;
    if (!out) out = si;
    out[0] = a; out[1] = b; return 1;
}

/* get_suffix (bwt.c:105-121) with FMindexCurrent (compactfmi.c:312-336) and
 * suffixArray_decode_number (suffixArray.h:37-51) */
void ko_get_suffix(const ko_index *x, int64_t i, int *iseq, int64_t *pos) {
    int64_t k = 0; int c = 1;
    while (c && (i & x->check)) { c = x->letters[i]; i = rank_(x, c, i); k++; }
    if (c) {
        int64_t e = (i >> x->chpt_exp) - ((int64_t)(x->nseq - 1) >> x->chpt_exp) - 1;
        /* The last sampled row of an index whose nseq is a multiple of 2^chpt_exp and whose bwtlen is not has no entry: the header counts one sample
         * less than kaiju-mkbwt writes (suffixArray.c:160 vs 206-216).  The reference decodes the bytes after its array there (heap
         * contents, often a sequence number >= nseq); the device reads its guard entry, "no taxon".  The oracle does as the device. */
        if (e >= x->ncheck) { *iseq = -1; *pos = -1; return; }
        const uint8_t *p = x->sa + e * x->nbytes; int64_t v = 0;
        for (int b = 0; b < x->nbytes; b++) v = (v << 8) + p[b];
        *iseq = (int)(v >> x->pbits); *pos = (v & x->mask) + k;
    } else { *iseq = (int)i; *pos = k - 1; }
}
static int get_suffix_counted(const ko_index *x, int64_t i, ko_counters *ctr) {
    int iseq; int64_t pos;
    if (ctr) { ctr->get_suffix++; int64_t j = i; int c = 1; while (c && (j & x->check)) { c = x->letters[j]; j = rank_(x, c, j); ctr->lf_steps++; } }
    ko_get_suffix(x, i, &iseq, &pos); return iseq;
}

/* ------------------------------------------------------------------------------------------
 * Taxonomy: parseNodesDmp (util.cpp:79-99) + lca_from_ids (util.cpp:194-263)
 * ------------------------------------------------------------------------------------------ */
struct ko_tax { uint64_t *key, *val; uint8_t *used; uint64_t cap, n; };
static uint64_t hmix(uint64_t k) { k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; return k; }
static void tax_put(ko_tax *t, uint64_t k, uint64_t v) {      /* unordered_map::emplace keeps the first */
    uint64_t i = hmix(k) & (t->cap - 1);
    while (t->used[i]) { if (t->key[i] == k) return; i = (i + 1) & (t->cap - 1); }
    t->used[i] = 1; t->key[i] = k; t->val[i] = v; t->n++;
}
static int tax_get(const ko_tax *t, uint64_t k, uint64_t *v) {
    uint64_t i = hmix(k) & (t->cap - 1);
    while (t->used[i]) { if (t->key[i] == k) { if (v) *v = t->val[i]; return 1; } i = (i + 1) & (t->cap - 1); }
    return 0;
}
ko_tax *ko_tax_load(const char *path) {
    FILE *fp = fopen(path, "r"); if (!fp) return NULL;
    size_t nl = 0; int ch; while ((ch = fgetc(fp)) != EOF) nl += (ch == '\n'); rewind(fp);
    ko_tax *t = (ko_tax *)calloc(1, sizeof(ko_tax));
    t->cap = 1024; while (t->cap < 2 * (nl + 16)) t->cap <<= 1;
    t->key = (uint64_t *)calloc(t->cap, 8); t->val = (uint64_t *)calloc(t->cap, 8); t->used = (uint8_t *)calloc(t->cap, 1);
    char line[4096];
    while (fgets(line, sizeof line, fp)) {
        const char *p = line; if (*p < '0' || *p > '9') continue;    /* stoul would throw -> line skipped */
        uint64_t node = strtoull(p, (char **)&p, 10);
        while (*p && (*p < '0' || *p > '9')) p++;
        if (!*p) continue;
        uint64_t parent = strtoull(p, NULL, 10);
        tax_put(t, node, parent);
    }
    fclose(fp); return t;
}
void ko_tax_free(ko_tax *t) { if (!t) return; free(t->key); free(t->val); free(t->used); free(t); }

uint64_t ko_lca(const ko_tax *t, const uint64_t *ids, int n) {
    if (n == 1) return ids[0];                                      /* util.cpp:197-199 */
    uint64_t leaf[64]; unsigned depth[64]; int m = 0; unsigned shallow = 100000;
    for (int i = 0; i < n && m < 64; i++) {
        if (!tax_get(t, ids[i], NULL)) continue;                    /* util.cpp:206-210 */
        unsigned d = 1; uint64_t id = ids[i], p;
        while (tax_get(t, id, &p) && p != id) { d++; id = p; }
        leaf[m] = ids[i]; depth[m] = d; if (d < shallow) shallow = d; m++;
    }
    if (m <= 0) return 0;
    for (int i = 0; i < m; i++) for (unsigned s = depth[i] - shallow; s > 0; s--) { uint64_t p = leaf[i]; tax_get(t, leaf[i], &p); leaf[i] = p; }
    for (int guard = 0; guard < 100000; guard++) {
        uint64_t first = leaf[0]; int same = 1;
        for (int i = 0; i < m; i++) { if (leaf[i] != first) same = 0; uint64_t p = leaf[i]; tax_get(t, leaf[i], &p); leaf[i] = p; }
        if (same) return first;
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * SEG (blast_seg.c).  Window 12, locut 2.2, hicut 2.5, maxtrim 50, maxbogus 2, overlaps TRUE.
 * Input restricted to the 20 standard residues (fragments never contain anything else), so
 * "bogus" is always 0 and H is never -1 inside [first,last].
 * ------------------------------------------------------------------------------------------ */
#define SEG_WINDOW 12
static const double SEG_LOCUT = 2.2, SEG_HICUT = 2.5;
#define SEG_MAXTRIM 50
#define KO_LNFACT_N 10001                /* entries of the reference table lnfact[0..10000] (blast_seg.c:53-1306) */
static double g_lnfact[KO_LNFACT_N]; static int g_lnfact_ready = 0;
double ko_lnfact(int n) {
    if (!g_lnfact_ready) {
        for (int i = 0; i < KO_LNFACT_N; i++) { char b[64]; snprintf(b, sizeof b, "%.6f", lgamma((double)i + 1.0)); g_lnfact[i] = strtod(b, NULL); }
        g_lnfact[0] = g_lnfact[1] = 0.0; g_lnfact_ready = 1;
    }
    if (n < KO_LNFACT_N) return g_lnfact[n];                        /* s_lnfact, blast_seg.c:1852-1856: table first */
    return ((n + 0.5) * log((double)n) - n + 0.9189385332);         /* s_lnfact, blast_seg.c:1852-1856 */
}
typedef struct { int begin, end; } seg_t;
typedef struct { seg_t *v; int n, cap; } seglist;                  /* index 0 = list head */
static void seglist_push_front(seglist *l, seg_t s) {
    if (l->n == l->cap) { l->cap = l->cap ? 2 * l->cap : 16; l->v = (seg_t *)realloc(l->v, sizeof(seg_t) * (size_t)l->cap); }
    memmove(l->v + 1, l->v, sizeof(seg_t) * (size_t)l->n); l->v[0] = s; l->n++;
}
/* sorted (descending) composition vector of s[0..len), zero terminated: s_CompOn/s_StateOn 1486-1546 */
static int state_vector(const char *s, int len, int *sv) {
    int comp[26]; memset(comp, 0, sizeof comp);
    for (int i = 0; i < len; i++) comp[s[i] - 'A']++;
    int n = 0; for (int a = 0; a < 26; a++) if (comp[a]) sv[n++] = comp[a];
    for (int i = 1; i < n; i++) { int v = sv[i], j = i; while (j > 0 && sv[j - 1] < v) { sv[j] = sv[j - 1]; j--; } sv[j] = v; }
    sv[n] = 0; return n;
}
static double seg_entropy(const int *sv) {                          /* s_Entropy 1596-1626 */
    int total = 0; for (int i = 0; sv[i]; i++) total += sv[i];
    if (!total) return 0.0;
    double ent = 0.0;
    for (int i = 0; sv[i]; i++) ent += ((double)sv[i]) * log(((double)sv[i]) / (double)total) / 0.69314718055994530941723212145818;
    return fabs(ent / (double)total);
}
static double seg_lnass(const int *sv) {                            /* s_LnAss 1890-1930, alphasize 20 */
    double ans = ko_lnfact(20);
    if (sv[0] == 0) return ans;
    int total = 20, cls = 1, i = 0, svi = sv[0], svim1 = sv[0];
    for (;; svim1 = svi) {
        if (++i == 20) { ans -= ko_lnfact(cls); break; }
        else if ((svi = sv[i]) == svim1) { cls++; continue; }
        else { total -= cls; ans -= ko_lnfact(cls); if (svi == 0) { ans -= ko_lnfact(total); break; } else { cls = 1; continue; } }
    }
    return ans;
}
static double seg_getprob(const int *sv, int total) {               /* s_GetProb 1941-1962 + s_LnPerm 1865-1879 */
    double totseq = ((double)total) * 2.9957322735539909;
    double ans1 = seg_lnass(sv), ans2 = 0;
    if (ans1 > -100000.0) { ans2 = ko_lnfact(total); for (int i = 0; sv[i]; i++) ans2 -= ko_lnfact(sv[i]); }
    return ans1 + ans2 - totseq;
}
static void seg_trim(const char *s, int n, int *leftend, int *rightend) {   /* s_Trim 1971-2015 */
    int lend = 0, rend = n - 1, minlen = 1;
    if (n - SEG_MAXTRIM > minlen) minlen = n - SEG_MAXTRIM;
    double minprob = 1.0; int sv[32];
    for (int len = n; len > minlen; len--)
        for (int i = 0; i + len <= n; i++) {
            state_vector(s + i, len, sv);
            double prob = seg_getprob(sv, len);
            if (prob < minprob) { minprob = prob; lend = i; rend = len + i - 1; }
        }
    *leftend += lend; *rightend -= (n - rend - 1);
}
static void seg_segseq(const char *s, int n, int offset, seglist *segs) {    /* s_SegSeq 2027-2113 */
    const int downset = (SEG_WINDOW + 1) / 2 - 1, upset = SEG_WINDOW - downset;
    if (SEG_WINDOW > n) return;
    double *H = (double *)malloc(sizeof(double) * (size_t)n);
    for (int i = 0; i < n; i++) H[i] = -1.0;
    int first = downset, last = n - upset, lowlim = first, sv[32];
    for (int i = first; i <= last; i++) { state_vector(s + i - downset, SEG_WINDOW, sv); H[i] = seg_entropy(sv); }   /* s_SeqEntropy 1751-1798 */
    for (int i = first; i <= last; i++) {
        if (H[i] <= SEG_LOCUT && H[i] != -1.0) {
            int loi, hii, j;
            for (j = i; j >= lowlim; j--) { if (H[j] == -1.0) break; if (H[j] > SEG_HICUT) break; } loi = j + 1;   /* s_FindLow */
            for (j = i; j <= last; j++) { if (H[j] == -1.0) break; if (H[j] > SEG_HICUT) break; } hii = j - 1;     /* s_FindHigh */
            int leftend = loi - downset, rightend = hii + upset - 1;
            seg_trim(s + leftend, rightend - leftend + 1, &leftend, &rightend);
            if (i + upset - 1 < leftend) {                           /* trigger window fell into the left trim */
                int lend = loi - downset, rend = leftend - 1;
                seglist left = {0, 0, 0};
                seg_segseq(s + lend, rend - lend + 1, offset + lend, &left);
                if (left.n > 0) seglist_push_front(segs, left.v[0]);   /* only the HEAD survives: 2093-2097 */
                free(left.v);
            }
            seg_t sg = { leftend + offset, rightend + offset };
            seglist_push_front(segs, sg);
            i = hii < rightend + downset ? hii : rightend + downset;
            lowlim = i + 1;
        }
    }
    free(H);
}
int ko_seg(const char *aa, int len, int *left, int *right, int max) {
    seglist segs = {0, 0, 0};
    seg_segseq(aa, len, 0, &segs);
    /* s_MergeSegs 2122-2152 with hilenmin 0, walking the list from its head */
    if (segs.n > 0) {
        int cur = 0;
        for (int nx = 1; nx < segs.n; ) {
            if (segs.v[cur].begin - segs.v[nx].end - 1 < 0) {
                if (segs.v[cur].end < segs.v[nx].end) segs.v[cur].end = segs.v[nx].end;
                if (segs.v[cur].begin > segs.v[nx].begin) segs.v[cur].begin = segs.v[nx].begin;
                memmove(segs.v + nx, segs.v + nx + 1, sizeof(seg_t) * (size_t)(segs.n - nx - 1)); segs.n--;
            } else { cur = nx; nx++; }
        }
    }
    /* s_SegsToBlastSeqLoc 2162-2180 prepends while walking -> reversed order */
    int n = 0;
    for (int i = segs.n - 1; i >= 0; i--) { if (n < max) { left[n] = segs.v[i].begin; right[n] = segs.v[i].end; } n++; }
    free(segs.v);
    return n;
}

/* ------------------------------------------------------------------------------------------
 * Fragments, queue, search drivers (ConsumerThread.cpp)
 * ------------------------------------------------------------------------------------------ */
static const char AA_ORDER[21] = "ARNDCQEGHILKMFPSTWYV";              /* aa2int, ConsumerThread.cpp:45-65 */
static int8_t g_diag[20], g_b62[20][20]; static uint8_t g_aa2int[256]; static char g_subst[26][20];
static uint8_t g_nuc[256], g_cnuc[256]; static char g_codon2aa[256]; static int g_tables = 0;
static const char *B62_ROWS[20] = {   /* BLOSUM62, rows/cols in AA_ORDER (values as ConsumerThread.cpp:66-107) */
 "4 -1 -2 -2 0 -1 -1 0 -2 -1 -1 -1 -1 -2 -1 1 0 -3 -2 0", "-1 5 0 -2 -3 1 0 -2 0 -3 -2 2 -1 -3 -2 -1 -1 -3 -2 -3",
 "-2 0 6 1 -3 0 0 0 1 -3 -3 0 -2 -3 -2 1 0 -4 -2 -3", "-2 -2 1 6 -3 0 2 -1 -1 -3 -4 -1 -3 -3 -1 0 -1 -4 -3 -3",
 "0 -3 -3 -3 9 -3 -4 -3 -3 -1 -1 -3 -1 -2 -3 -1 -1 -2 -2 -1", "-1 1 0 0 -3 5 2 -2 0 -3 -2 1 0 -3 -1 0 -1 -2 -1 -2",
 "-1 0 0 2 -4 2 5 -2 0 -3 -3 1 -2 -3 -1 0 -1 -3 -2 -2", "0 -2 0 -1 -3 -2 -2 6 -2 -4 -4 -2 -3 -3 -2 0 -2 -2 -3 -3",
 "-2 0 1 -1 -3 0 0 -2 8 -3 -3 -1 -2 -1 -2 -1 -2 -2 2 -3", "-1 -3 -3 -3 -1 -3 -3 -4 -3 4 2 -3 1 0 -3 -2 -1 -3 -1 3",
 "-1 -2 -3 -4 -1 -2 -3 -4 -3 2 4 -2 2 0 -3 -2 -1 -2 -1 1", "-1 2 0 -1 -3 1 1 -2 -1 -3 -2 5 -1 -3 -1 0 -1 -3 -2 -2",
 "-1 -1 -2 -3 -1 0 -2 -3 -2 1 2 -1 5 0 -2 -1 -1 -1 -1 1", "-2 -3 -3 -3 -2 -3 -3 -3 -1 0 0 -3 0 6 -4 -2 -2 1 3 -1",
 "-1 -2 -2 -1 -3 -1 -1 -2 -2 -3 -3 -1 -2 -4 7 -1 -1 -4 -3 -2", "1 -1 1 0 -1 0 0 0 -1 -2 -2 0 -1 -2 -1 4 1 -3 -2 -2",
 "0 -1 0 -1 -1 -1 -1 -2 -2 -1 -1 -1 -1 -2 -1 1 5 -2 -2 0", "-3 -3 -4 -4 -2 -2 -3 -2 -2 -3 -2 -3 -1 1 -4 -3 -2 11 2 -3",
 "-2 -2 -2 -3 -2 -1 -2 -3 2 -1 -1 -2 -1 3 -3 -2 -2 2 7 -1", "0 -3 -3 -3 -1 -2 -2 -3 -3 3 1 -2 1 -1 -2 -2 0 -3 -1 4" };
/* substitution try-order per residue (ConsumerThread.cpp:10-30), keyed by the residue letter */
static const char *SUBST_ORDER[20] = {
 "A:SVTGCPMKLIEQRYFHDNW", "R:KQHENTSMAYPLGDVWFIC", "N:SHDTKGEQRYPMAVFLICW", "D:ENSQTPKHGRAVYFMICWL", "C:AVTSMLIYWFPKHGQDNRE",
 "Q:EKRSMHDNYTPAVWLGFIC", "E:QDKSHNRTPAVYMGWFLIC", "G:SNADWTPKHEQRVYFMCLI", "H:YNEQRSFKDWTPMGAVLIC", "I:VLMFYTCASWPKHEQDNRG",
 "L:MIVFYTCAWSKQRPHENGD", "K:REQSNTPMHDAVYLGWFIC", "M:LVIFQYWTSKCRAPHENGD", "F:YWMLIVHTSCAKGEQDNRP", "P:TSKEQDAVMHGNRYLICWF",
 "S:TNAKGEQDPMHCRVYFLIW", "T:SVNAPMKLIEQCDRYWFHG", "W:YFMTLHGQCVSKIERAPDN", "Y:FWHVMLIQTSKECNRAPGD", "V:IMLTAYFCSPKEQWHGDNR" };
static void init_tables(void) {
    if (g_tables) return;
    memset(g_aa2int, 0, sizeof g_aa2int);
    for (int i = 0; i < 20; i++) g_aa2int[(uint8_t)AA_ORDER[i]] = (uint8_t)i;
    for (int i = 0; i < 20; i++) { const char *p = B62_ROWS[i]; for (int j = 0; j < 20; j++) { g_b62[i][j] = (int8_t)strtol(p, (char **)&p, 10); } g_diag[i] = g_b62[i][i]; }
    for (int i = 0; i < 20; i++) memcpy(g_subst[SUBST_ORDER[i][0] - 'A'], SUBST_ORDER[i] + 2, 19);
    memset(g_nuc, 255, 256); memset(g_cnuc, 255, 256);                    /* ConsumerThread.cpp:32-43 */
    g_nuc['A'] = g_nuc['a'] = 0; g_nuc['C'] = g_nuc['c'] = 1; g_nuc['G'] = g_nuc['g'] = 2; g_nuc['T'] = g_nuc['t'] = 3; g_nuc['U'] = g_nuc['u'] = 3;
    g_cnuc['A'] = g_cnuc['a'] = 3; g_cnuc['C'] = g_cnuc['c'] = 2; g_cnuc['G'] = g_cnuc['g'] = 1; g_cnuc['T'] = g_cnuc['t'] = 0; g_cnuc['U'] = g_cnuc['u'] = 0;
    /* standard genetic code, index = n0<<4|n1<<2|n2 with A0 C1 G2 T3 (ConsumerThread.cpp:117-181) */
    static const char code[65] = "KNKNTTTTRSRSIIMIQHQHPPPPRRRRLLLLEDEDAAAAGGGGVVVV*Y*YSSSS*CWCLFLF";
    memset(g_codon2aa, '*', 256); memcpy(g_codon2aa, code, 64);
    g_tables = 1;
}
static inline int diag_of(char c) { return g_diag[g_aa2int[(uint8_t)c]]; }

typedef struct {
    char *seq; int len; unsigned num_mm; int diff; int64_t si0, si1; int matchlen; int segchecked;
    unsigned key; uint64_t order;
} frag_t;
typedef struct { frag_t *v; int n, cap; uint64_t next_order; } fragq;    /* std::multimap<unsigned,Fragment*,greater> */
static void fq_push(fragq *q, unsigned key, const char *s, int len, unsigned num_mm, int diff, int64_t si0, int64_t si1, int matchlen, int segchecked) {
    if (q->n == q->cap) { q->cap = q->cap ? q->cap * 2 : 64; q->v = (frag_t *)realloc(q->v, sizeof(frag_t) * (size_t)q->cap); }
    frag_t *f = &q->v[q->n++];
    f->seq = (char *)malloc((size_t)len + 1); memcpy(f->seq, s, (size_t)len); f->seq[len] = 0; f->len = len;
    f->num_mm = num_mm; f->diff = diff; f->si0 = si0; f->si1 = si1; f->matchlen = matchlen; f->segchecked = segchecked;
    f->key = key; f->order = q->next_order++;
}
static int fq_top(const fragq *q) {                 /* highest key, FIFO among equal keys */
    int b = -1;
    for (int i = 0; i < q->n; i++) if (b < 0 || q->v[i].key > q->v[b].key || (q->v[i].key == q->v[b].key && q->v[i].order < q->v[b].order)) b = i;
    return b;
}
static frag_t fq_take(fragq *q, int i) { frag_t f = q->v[i]; q->v[i] = q->v[--q->n]; return f; }
static void fq_clear(fragq *q) { for (int i = 0; i < q->n; i++) free(q->v[i].seq); q->n = 0; q->next_order = 0; }

static unsigned self_score(const char *s, int len) { unsigned sc = 0; for (int i = 0; i < len; i++) sc += (unsigned)diag_of(s[i]); return sc; }   /* calcScore(s), 415-421 */
static unsigned calc_score(const char *s, int start, int len, int diff) {        /* calcScore(s,start,len,diff), 397-404 */
    int sc = 0; for (int i = start; i < start + len; i++) sc += diag_of(s[i]); sc += diff; return sc > 0 ? (unsigned)sc : 0u;
}
static void emit_fragment(fragq *q, const ko_params *P, const char *s, int len, int segchecked, ko_counters *ctr) {
    if (P->mode == 1) { unsigned sc = self_score(s, len); if (sc >= P->min_score) fq_push(q, sc, s, len, 0, 0, 0, 0, 0, segchecked); else return; }
    else fq_push(q, (unsigned)len, s, len, 0, 0, 0, 0, 0, segchecked);
    if (ctr && !segchecked) ctr->fragments_initial++;
}
/* getAllFragmentsBits (ConsumerThread.cpp:190-270) */
static void all_fragments(fragq *q, const ko_params *P, const char *line, int n, ko_counters *ctr) {
    char *tr[3]; int tl[3] = {0, 0, 0};
    for (int f = 0; f < 3; f++) tr[f] = (char *)malloc((size_t)n / 3 + 4);
    const unsigned m = P->min_fragment_length;
    for (int count = 0; count + 2 < n; count++) {
        uint8_t ci = (uint8_t)(g_nuc[(uint8_t)line[count]] << 4 | g_nuc[(uint8_t)line[count + 1]] << 2 | g_nuc[(uint8_t)line[count + 2]]);
        char aa = g_codon2aa[ci]; int f = count % 3;
        if (aa == '*') { if ((unsigned)tl[f] >= m) emit_fragment(q, P, tr[f], tl[f], 0, ctr); tl[f] = 0; }
        else tr[f][tl[f]++] = aa;
    }
    for (int f = 0; f < 3; f++) { if ((unsigned)tl[f] >= m) emit_fragment(q, P, tr[f], tl[f], 0, ctr); tl[f] = 0; }
    /* reverse strand: the first iteration (count = n-2) reads the NUL terminator -> '*' on empty buffers */
    for (int count = n - 3; count >= 0; count--) {
        uint8_t ci = (uint8_t)(g_cnuc[(uint8_t)line[count + 2]] << 4 | g_cnuc[(uint8_t)line[count + 1]] << 2 | g_cnuc[(uint8_t)line[count]]);
        char aa = g_codon2aa[ci]; int f = count % 3;
        if (aa == '*') { if ((unsigned)tl[f] >= m) emit_fragment(q, P, tr[f], tl[f], 0, ctr); tl[f] = 0; }
        else tr[f][tl[f]++] = aa;
    }
    for (int f = 0; f < 3; f++) { if ((unsigned)tl[f] >= m) emit_fragment(q, P, tr[f], tl[f], 0, ctr); }
    for (int f = 0; f < 3; f++) free(tr[f]);
}
int ko_fragments(const char *seq, int len, int min_len, char *buf, int bufsize) {
    init_tables();
    ko_params P; memset(&P, 0, sizeof P); P.mode = 0; P.min_fragment_length = (uint32_t)min_len;
    fragq q = {0, 0, 0, 0}; if (len >= 3) all_fragments(&q, &P, seq, len, NULL);
    /* insertion order */
    int o = 0, cnt = 0;
    for (uint64_t ord = 0; ord < q.next_order; ord++) for (int i = 0; i < q.n; i++) if (q.v[i].order == ord) {
        if (o + q.v[i].len + 1 <= bufsize) { memcpy(buf + o, q.v[i].seq, (size_t)q.v[i].len + 1); o += q.v[i].len + 1; cnt++; }
    }
    fq_clear(&q); free(q.v); return cnt;
}

/* getNextFragment (ConsumerThread.cpp:272-342): pop + lazy SEG */
static int next_fragment(fragq *q, const ko_params *P, unsigned min_key, frag_t *out, ko_counters *ctr) {
    int t = fq_top(q); if (t < 0) return 0;
    if (q->v[t].key < min_key) return 0;
    frag_t f = fq_take(q, t);
    while (P->seg && !f.segchecked) {
        enum { KO_SEG_MAXREG = 8192 }; static __thread int L[KO_SEG_MAXREG], R[KO_SEG_MAXREG]; if (ctr) ctr->seg_calls++;
        int ns = ko_seg(f.seq, f.len, L, R, KO_SEG_MAXREG);
        if (ns > 0) {
            if (ctr) ctr->seg_hits++;
            int start = 0;
            for (int s = 0; s < ns; s++) {
                int length = L[s] - start;            /* size_t arithmetic in the reference; L[s] >= start always */
                if (length > (int)P->min_fragment_length) emit_fragment(q, P, f.seq + start, length, 1, ctr);
                start = R[s] + 1;
            }
            int lastlen = f.len - start;
            if (lastlen > (int)P->min_fragment_length) emit_fragment(q, P, f.seq + start, lastlen, 1, ctr);
            free(f.seq);
            t = fq_top(q); if (t < 0) return 0;
            if (q->v[t].key >= min_key) f = fq_take(q, t); else return 0;
        } else break;
    }
    *out = f; return 1;
}

typedef struct { int64_t start; int len, qi, ql; } si_t;            /* SI, bwt.h:25-34 */
typedef struct { si_t *v; int n, cap; } silist;
static void sl_push(silist *l, si_t s) { if (l->n == l->cap) { l->cap = l->cap ? 2 * l->cap : 32; l->v = (si_t *)realloc(l->v, sizeof(si_t) * (size_t)l->cap); } l->v[l->n++] = s; }

/* backward extension from j: returns match start i and the interval (the inner loop of bwt.c:267-275) */
static int extend_from(const ko_index *x, const uint8_t *str, int j, int64_t si[2], ko_counters *ctr) {
    int i = j; initial_si(x, str[i], si, ctr);
    while (i-- > 0) { if (!update_si(x, str[i], si, NULL, ctr)) break; }
    return i + 1;
}
/* greedyExact(f,str,len,L,-1) (bwt.c:347-380): out = samelen chain, head first */
static void greedy_exact(const ko_index *x, const uint8_t *str, int len, int L, silist *out, ko_counters *ctr) {
    out->n = 0;
    silist tmp = {0, 0, 0};                                          /* found order */
    for (int j = len - 1; j >= L - 1; j--) {
        int64_t si[2]; int i = extend_from(x, str, j, si, ctr); int l = j - i + 1;
        if (l >= L) { if (l > L) { tmp.n = 0; L = l; } si_t s = { si[0], (int)(si[1] - si[0]), i, l }; sl_push(&tmp, s); }
        if (i <= 1) break;
    }
    for (int k = tmp.n - 1; k >= 0; k--) sl_push(out, tmp.v[k]);    /* newest is the head */
    free(tmp.v);
}
/* maxMatches(f,str,len,L,0) (bwt.c:261-296) with insert_SI_sorted (225-252).
 * Result: classes sorted by ql descending; cls_start[c]..cls_start[c+1] index into out->v where each
 * class is stored in FOUND order (f1,f2,..,fn); the reference's samelen chain is f1,fn,..,f2. */
static int max_matches(const ko_index *x, const uint8_t *str, int len, int L, silist *out, int *cls_start, ko_counters *ctr) {
    silist found = {0, 0, 0}; int have_cur = 0, cur_qi = 0;
    for (int j = len - 1; j >= L - 1; j--) {
        int64_t si[2]; int i = extend_from(x, str, j, si, ctr); int l = j - i + 1;
        if (l >= L && (!have_cur || i < cur_qi)) { si_t s = { si[0], (int)(si[1] - si[0]), i, l }; sl_push(&found, s); have_cur = 1; cur_qi = i; }
        if (i <= 1) break;
    }
    out->n = 0; int ncls = 0;
    /* distinct lengths, descending */
    int *lens = (int *)malloc(sizeof(int) * (size_t)(found.n + 1)), nl = 0;
    for (int k = 0; k < found.n; k++) { int seen = 0; for (int t = 0; t < nl; t++) if (lens[t] == found.v[k].ql) seen = 1; if (!seen) lens[nl++] = found.v[k].ql; }
    for (int a = 1; a < nl; a++) { int v = lens[a], b = a; while (b > 0 && lens[b - 1] < v) { lens[b] = lens[b - 1]; b--; } lens[b] = v; }
    for (int t = 0; t < nl; t++) { cls_start[ncls++] = out->n; for (int k = 0; k < found.n; k++) if (found.v[k].ql == lens[t]) sl_push(out, found.v[k]); }
    cls_start[ncls] = out->n;
    free(found.v); free(lens); return ncls;
}
/* maxMatches_withStart (bwt.c:298-336) */
static int max_matches_with_start(const ko_index *x, const uint8_t *str, int len, int L, int64_t si0, int64_t si1, int offset, si_t *out, ko_counters *ctr) {
    int64_t si[2] = { si0, si1 }; int j = len - 1, i = j - offset + 1;
    while (i-- > 0) { if (!update_si(x, str[i], si, NULL, ctr)) break; }
    i += 1; int l = j - i + 1;
    if (l >= L) { out->start = si[0]; out->len = (int)(si[1] - si[0]); out->qi = i; out->ql = l; return 1; }
    return 0;
}

typedef struct { uint64_t v[64]; int n; } idset;                   /* std::set<uint64_t> match_ids */
static void ids_insert(idset *s, uint64_t id) {
    int i = 0; while (i < s->n && s->v[i] < id) i++;
    if (i < s->n && s->v[i] == id) return;
    if (s->n >= 64) return;
    memmove(s->v + i + 1, s->v + i, sizeof(uint64_t) * (size_t)(s->n - i)); s->v[i] = id; s->n++;
}
/* ids_from_SI (ConsumerThread.cpp:799-835), max_match_ids = 20 */
static void ids_from_si(const ko_index *x, const si_t *s, idset *ids, ko_counters *ctr) {
    for (int64_t k = s->start; k < s->start + s->len; k++) {
        if (ids->n > 20) break;
        int iseq = get_suffix_counted(x, k, ctr);
        if (iseq < 0) continue;                                    /* the guard row (ko_get_suffix) */
        uint64_t id = x->seq_taxon[iseq];
        if (id == ULONG_MAX) continue;
        ids_insert(ids, id);
    }
}

/* classify_length (ConsumerThread.cpp:543-628) */
static uint64_t classify_length(const ko_index *x, const ko_tax *T, const ko_params *P, fragq *q, uint32_t *best, idset *ids, ko_counters *ctr) {
    unsigned longest = 0; silist kept = {0, 0, 0}, chain = {0, 0, 0}; frag_t t;
    while (next_fragment(q, P, longest, &t, ctr)) {
        uint8_t *num = (uint8_t *)malloc((size_t)t.len + 1);
        for (int i = 0; i < t.len; i++) num[i] = x->trans[(uint8_t)t.seq[i]];              /* translate2numbers */
        if (ctr) ctr->fragments_searched++;
        unsigned L = P->min_fragment_length > longest ? P->min_fragment_length : longest;
        greedy_exact(x, num, t.len, (int)L, &chain, ctr);
        if (chain.n > 0) {
            unsigned ql = (unsigned)chain.v[0].ql;
            if (ql > longest) { kept.n = 0; longest = ql; for (int k = 0; k < chain.n; k++) sl_push(&kept, chain.v[k]); }
            else if (ql == longest) { for (int k = 0; k < chain.n; k++) sl_push(&kept, chain.v[k]); }
        }
        free(num); free(t.seq);
    }
    ids->n = 0; uint64_t lca = 0; *best = 0;
    if (kept.n > 0) {
        for (int k = 0; k < kept.n; k++) ids_from_si(x, &kept.v[k], ids, ctr);            /* ids_from_SI_recursive 837-845 */
        *best = longest;
        lca = ids->n == 1 ? ids->v[0] : ko_lca(T, ids->v, ids->n);
    }
    free(kept.v); free(chain.v);
    return lca;
}

/* addAllMismatchVariantsAtPosSI (ConsumerThread.cpp:346-395) */
static void add_variants(const ko_index *x, const ko_params *P, fragq *q, const frag_t *f, int pos, int erase_pos, const si_t *si, unsigned best, ko_counters *ctr) {
    int len = f->len; if (erase_pos >= 0 && erase_pos < len) len = erase_pos;
    char *fr = (char *)malloc((size_t)len + 1); memcpy(fr, f->seq, (size_t)len); fr[len] = 0;
    char orig = fr[pos]; int oi = g_aa2int[(uint8_t)orig];
    int score = (int)calc_score(fr, 0, len, f->diff) - g_diag[oi];
    int64_t sia[2] = { si->start, si->start + si->len }, upd[2];
    const char *order = g_subst[orig - 'A'];
    for (int k = 0; k < 19; k++) {
        char sub = order[k]; int sj = g_aa2int[(uint8_t)sub];
        int after = score + g_b62[oi][sj];
        if (after >= (int)best && after >= (int)P->min_score) {
            if (update_si(x, x->trans[(uint8_t)sub], sia, upd, ctr)) {
                fr[pos] = sub;
                int d = g_b62[oi][sj] - g_diag[sj];
                fq_push(q, (unsigned)after, fr, len, f->num_mm + 1, f->diff + d, upd[0], upd[1], si->ql + 1, 1);
            }
        } else break;
    }
    free(fr);
}

typedef struct { si_t v[32]; int n; unsigned best; } bestlist;
static void score_one(const ko_params *P, const frag_t *t, const si_t *s, bestlist *B) {      /* tail of eval_match_scores 763-794 */
    unsigned sc = calc_score(t->seq, s->qi, s->ql, t->diff);
    if (sc < P->min_score) return;
    if (sc > B->best) { B->n = 0; B->v[B->n++] = *s; B->best = sc; }
    else if (sc == B->best && B->n < 20) B->v[B->n++] = *s;
}
/* eval_match_scores (751-797) over classes [c..ncls): samelen chain first (f2..fn), then the next class
 * if its ql >= m, then the class head f1. */
static void eval_classes(const ko_params *P, const frag_t *t, const silist *S, const int *cls, int c, int ncls, bestlist *B) {
    if (c >= ncls) return;
    for (int k = cls[c] + 1; k < cls[c + 1]; k++) score_one(P, t, &S->v[k], B);
    if (c + 1 < ncls && S->v[cls[c + 1]].ql >= (int)P->min_fragment_length) eval_classes(P, t, S, cls, c + 1, ncls, B);
    score_one(P, t, &S->v[cls[c]], B);
}

/* classify_greedyblosum (ConsumerThread.cpp:424-541) */
static uint64_t classify_greedy(const ko_index *x, const ko_tax *T, const ko_params *P, fragq *q, double query_len, uint32_t *best, idset *ids, ko_counters *ctr) {
    bestlist B; B.n = 0; B.best = 0; frag_t t; silist S = {0, 0, 0};
    while (next_fragment(q, P, B.best, &t, ctr)) {
        uint8_t *num = (uint8_t *)malloc((size_t)t.len + 1);
        for (int i = 0; i < t.len; i++) num[i] = x->trans[(uint8_t)t.seq[i]];
        if (ctr) ctr->fragments_searched++;
        int ncls = 0; int *cls = (int *)malloc(sizeof(int) * (size_t)(t.len + 2));   /* class boundaries: at most one class per match length */
        if (t.num_mm > 0) {
            si_t one; int L = (t.num_mm == P->mismatches) ? (int)P->min_fragment_length : t.matchlen;
            S.n = 0;
            if (max_matches_with_start(x, num, t.len, L, t.si0, t.si1, t.matchlen, &one, ctr)) { sl_push(&S, one); cls[0] = 0; cls[1] = 1; ncls = 1; }
        } else ncls = max_matches(x, num, t.len, (int)P->seed_length, &S, cls, ctr);
        if (ncls > 0) {
            if (P->mismatches > 0 && t.num_mm < P->mismatches) {
                /* walk: head; then its samelen chain (fn..f2) if it has one, else the next class head */
                int c = 0;
                while (c < ncls) {
                    int nmem = cls[c + 1] - cls[c];
                    for (int w = 0; w < nmem; w++) {
                        const si_t *s = (w == 0) ? &S.v[cls[c]] : &S.v[cls[c + 1] - w];
                        int mre = s->qi + s->ql - 1;
                        if (s->qi > 0 && (unsigned)(mre + 1) >= P->min_fragment_length)
                            add_variants(x, P, q, &t, s->qi - 1, (mre < t.len - 1) ? mre + 1 : -1, s, B.best, ctr);
                    }
                    if (nmem > 1) break;                              /* samelen nodes have next == NULL */
                    c++;
                }
            }
            if (S.v[cls[0]].ql >= (int)P->min_fragment_length) eval_classes(P, &t, &S, cls, 0, ncls, &B);
        }
        free(num); free(t.seq); free(cls);
    }
    free(S.v);
    ids->n = 0; *best = 0;
    if (B.n == 0) return 0;
    if (P->use_evalue) {                                             /* 500-513, constants ConsumerThread.hpp:41-44 */
        double bitscore = (0.3176 * B.best - (-2.009915479)) / 0.6931471805;
        double db_length = (double)(x->len - x->nseq);               /* Config.cpp:20 */
        double E = db_length * query_len * pow(2, -1 * bitscore);
        if (E > P->min_evalue) return 0;
    }
    for (int k = 0; k < B.n; k++) ids_from_si(x, &B.v[k], ids, ctr);
    *best = B.best;
    return ids->n == 1 ? ids->v[0] : ko_lca(T, ids->v, ids->n);
}

/* ConsumerThread::doWork body for one item (630-749) */
uint64_t ko_classify(const ko_index *x, const ko_tax *T, const ko_params *P, const char *seq1, int len1, const char *seq2, int len2,
                     uint32_t *best, uint64_t *ids_out, int *n_ids_out, ko_counters *ctr) {
    init_tables();
    uint32_t b = 0; idset ids; ids.n = 0; uint64_t lca = 0;
    const unsigned m = P->min_fragment_length; int paired = seq2 != NULL;
    if (ctr) { ctr->reads++; ctr->bases += (uint64_t)len1 + (uint64_t)(paired ? len2 : 0); }
    fragq q = {0, 0, 0, 0}; double query_len; int skip = 0;
    if (P->input_is_protein) {                                       /* 640-646, 659-696 */
        if ((unsigned)len1 < m) skip = 1;
        else {
            query_len = (double)len1; int start = 0; char *up = (char *)malloc((size_t)len1 + 1);
            for (int i = 0; i < len1; i++) { char c = seq1[i]; up[i] = (c >= 'a' && c <= 'z') ? (char)(c - 32) : c; }
            for (int pos = 0; pos <= len1; pos++) {
                int valid = pos < len1 && strchr("ACDEFGHIKLMNPQRSTVWY", up[pos]) != NULL && up[pos] != 0;
                if (!valid) { if ((unsigned)(pos - start) >= m) emit_fragment(&q, P, up + start, pos - start, 0, ctr); start = pos + 1; }
            }
            free(up);
        }
    } else {
        if ((!paired && (unsigned)len1 < m * 3) || (paired && (unsigned)len1 < m * 3 && (unsigned)len2 < m * 3)) skip = 1;   /* 648-653 */
        else {
            query_len = (double)len1 / 3.0;
            if ((unsigned)len1 >= m * 3) all_fragments(&q, P, seq1, len1, ctr);
            if (paired) { query_len += (double)len2 / 3.0; if ((unsigned)len2 >= m * 3) all_fragments(&q, P, seq2, len2, ctr); }
        }
    }
    if (!skip) {
        if (P->mode == 0) lca = classify_length(x, T, P, &q, &b, &ids, ctr);
        else lca = classify_greedy(x, T, P, &q, query_len, &b, &ids, ctr);
    }
    fq_clear(&q); free(q.v);
    if (ctr && lca) ctr->classified++;
    if (best) *best = lca ? b : 0;
    if (ids_out) { for (int i = 0; i < ids.n && i < 32; i++) ids_out[i] = ids.v[i]; }
    if (n_ids_out) *n_ids_out = ids.n;
    return lca;
}

void ko_classify_batch(const ko_index *x, const ko_tax *T, const ko_params *P, const char *seq1, const uint64_t *off1,
                       const char *seq2, const uint64_t *off2, uint64_t n, uint64_t *taxon_out, uint32_t *best_out, ko_counters *ctr) {
    for (uint64_t i = 0; i < n; i++) {
        uint32_t b = 0;
        /* the reference works on NUL-terminated std::string; make terminated copies */
        int l1 = (int)(off1[i + 1] - off1[i]), l2 = seq2 ? (int)(off2[i + 1] - off2[i]) : 0;
        char *a = (char *)malloc((size_t)l1 + 1); memcpy(a, seq1 + off1[i], (size_t)l1); a[l1] = 0;
        char *c = NULL; if (seq2) { c = (char *)malloc((size_t)l2 + 1); memcpy(c, seq2 + off2[i], (size_t)l2); c[l2] = 0; }
        taxon_out[i] = ko_classify(x, T, P, a, l1, c, l2, &b, NULL, NULL, ctr);
        if (best_out) best_out[i] = b;
        free(a); free(c);
    }
}
