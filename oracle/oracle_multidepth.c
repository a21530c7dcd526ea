/* oracle_multidepth.c — TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * A literal restatement of `goleft multidepth` (multidepth/multidepth.go) over per-base depth arrays, site by site:
 *   - a site is a position where at least one sample has depth > 0 (a line of `samtools depth` without -a);
 *   - minSamples = int(0.5 + MinSamples * S) (main, :64); sufficient = #samples with d >= MinCov is > minSamples (:158-166);
 *   - chunks: chunkSize = 5e6, / 5 when S > 50 (:60-62, :121); chunk k reads [k*C, contig end) (`-r chrom:k*C+1`, :126-138);
 *   - aggregate (:208-266): seen0, the kill test (pos0 > start1 + C and (empty cache or pos0 - last >= MaxSkip)), chaining
 *     (pos0 - (last + 1) <= MaxSkip), MinSize on a broken chain only, the cache left at the kill / contig end flushed as is;
 *   - splitBlocks (:183-200): a new block at the first cached site with pos0 - blockstart >= Window;
 *   - means (:268-283): acc += float64(d)/1000. in position order, acc/float64(l)*1000 with l the span, printed "%.2f".
 * Chunks are written in chunk order (the reference with -p 1).
 * Build flags: -ffp-contract=off (no FMA: Go on amd64 rounds every operation).
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

typedef struct { int64_t *v; int64_t n, cap; } ivec;

static void iv_push(ivec* a, int64_t x) {
    if (a->n == a->cap) {
        a->cap = a->cap ? 2 * a->cap : 1024;
        a->v = (int64_t*)realloc(a->v, (size_t)a->cap * sizeof(int64_t));
    }
    a->v[a->n++] = x;
}

/* blocks out: triples (start, end, first cached-site index into `sites`), sites = every cached site of every block */
typedef struct { ivec blk; ivec sites; } md_out;

static void split_blocks(md_out* o, const int64_t* cache, int64_t n, int64_t window) {
    int64_t i = 0;
    while (i < n) {
        const int64_t start = cache[i];
        const int64_t first = i;
        i++;
        for (; i < n && cache[i] - start < window; i++) {}
        iv_push(&o->blk, start);
        iv_push(&o->blk, cache[i - 1] + 1);
        iv_push(&o->blk, o->sites.n);
        for (int64_t k = first; k < i; k++) iv_push(&o->sites, cache[k]);
    }
}

int64_t orc_md_chunk_size(int64_t S) { return S > 50 ? 5000000 / 5 : 5000000; }
int64_t orc_md_min_samples(double frac, int64_t S) { return (int64_t)(0.5 + frac * (double)S); }

/* cls[x]: 0 = not a site, 1 = insufficient site, 2 = sufficient site */
static void aggregate_all(const uint8_t* cls, int64_t L, int64_t C, int64_t max_skip, int64_t min_size, int64_t window, md_out* o) {
    ivec cache = {0, 0, 0};
    for (int64_t k0 = 0; k0 < L; k0 += C) {
        const int64_t start1 = k0 + 1;
        cache.n = 0;
        int seen0 = 0;
        for (int64_t pos0 = k0; pos0 < L; pos0++) {
            if (cls[pos0] == 0) continue;
            const int suf = cls[pos0] == 2;
            if (!suf) {
                seen0 = 1;
                if (pos0 > start1 + C) {
                    if (cache.n == 0 || pos0 - cache.v[cache.n - 1] >= max_skip) break;
                }
            }
            if (!seen0) continue;
            if ((cache.n == 0 || pos0 - (cache.v[cache.n - 1] + 1) <= max_skip) && suf) {
                iv_push(&cache, pos0);
            } else if (cache.n > 0 && pos0 - (cache.v[cache.n - 1] + 1) > max_skip) {
                if (cache.n >= min_size) split_blocks(o, cache.v, cache.n, window);
                cache.n = 0;
                if (suf) iv_push(&cache, pos0);
            }
        }
        if (cache.n > 0) split_blocks(o, cache.v, cache.n, window);
    }
    free(cache.v);
}

/* Blocks from a site-class array.  out3 (may be NULL) gets (start, end, number of sites) per block; returns the block count. */
int64_t orc_md_blocks(const uint8_t* cls, int64_t L, int64_t C, int64_t max_skip, int64_t min_size, int64_t window,
                      int64_t* out3, int64_t cap) {
    md_out o;
    memset(&o, 0, sizeof o);
    aggregate_all(cls, L, C, max_skip, min_size, window, &o);
    const int64_t nb = o.blk.n / 3;
    for (int64_t b = 0; b < nb && b < cap && out3; b++) {
        const int64_t s0 = o.blk.v[3 * b + 2], s1 = b + 1 < nb ? o.blk.v[3 * b + 5] : o.sites.n;
        out3[3 * b] = o.blk.v[3 * b];
        out3[3 * b + 1] = o.blk.v[3 * b + 1];
        out3[3 * b + 2] = s1 - s0;
    }
    free(o.blk.v);
    free(o.sites.v);
    return nb;
}

/* The means of one block, as the reference computes them: sites = the block's positions, depth = one sample's array. */
double orc_md_mean(const int32_t* depth, const int64_t* sites, int64_t n) {
    double acc = 0;
    for (int64_t i = 0; i < n; i++) acc += (double)depth[sites[i]] / 1000.;
    const int64_t l = sites[n - 1] - sites[0] + 1;
    return acc / (double)l * 1000;
}

/* The same chain for a block given as "every position in [s, e) with bit set in suf" (the library's walk). */
double orc_md_mean_masked(const int32_t* depth, const uint8_t* suf, int64_t s, int64_t e) {
    double acc = 0;
    for (int64_t x = s; x < e; x++)
        if (suf[x]) acc += (double)depth[x] / 1000.;
    return acc / (double)(e - s) * 1000;
}

/* Sequential chain over n given depths spread over a span l (certification tests): acc += d/1000., acc/l*1000. */
double orc_md_chain(const int32_t* d, int64_t n, int64_t l) {
    double acc = 0;
    for (int64_t i = 0; i < n; i++) acc += (double)d[i] / 1000.;
    return acc / (double)l * 1000;
}

/* "%.2f" of a double into buf (returns the length) */
int orc_md_fmt2(double v, char* buf, int cap) { return snprintf(buf, (size_t)cap, "%.2f", v); }

/* The whole tool on depth arrays: depth = S rows of L int32 (row-major).  Writes the rows after the header line into a
 * malloc'd buffer (*text, *len; release with orc_free).  chunk = 0: the reference's chunk size for S samples.
 * Also returns the site classes when cls_out != NULL. */
int orc_md_text(const char* chrom, const int32_t* depth, int64_t S, int64_t L, int64_t mincov, double min_samples,
                int64_t max_skip, int64_t min_size, int64_t window, int64_t chunk, uint8_t* cls_out, char** text, int64_t* len) {
    const int64_t ms = orc_md_min_samples(min_samples, S);
    const int64_t C = chunk > 0 ? chunk : orc_md_chunk_size(S);
    uint8_t* cls = (uint8_t*)malloc((size_t)(L > 0 ? L : 1));
    for (int64_t x = 0; x < L; x++) {
        int64_t any = 0, n = 0;
        for (int64_t s = 0; s < S; s++) {
            const int32_t d = depth[s * L + x];
            any |= d > 0;
            n += d >= mincov;
        }
        cls[x] = !any ? 0 : (n > ms ? 2 : 1);
    }
    if (cls_out) memcpy(cls_out, cls, (size_t)L);
    md_out o;
    memset(&o, 0, sizeof o);
    aggregate_all(cls, L, C, max_skip, min_size, window, &o);
    const int64_t nb = o.blk.n / 3;
    size_t cap = 1 << 16, n = 0;
    char* out = (char*)malloc(cap);
    char tmp[64];
    for (int64_t b = 0; b < nb; b++) {
        const int64_t s0 = o.blk.v[3 * b + 2], s1 = b + 1 < nb ? o.blk.v[3 * b + 5] : o.sites.n;
        for (;;) {
            size_t need = strlen(chrom) + 48 + (size_t)S * 48;
            if (n + need < cap) break;
            cap *= 2;
            out = (char*)realloc(out, cap);
        }
        n += (size_t)sprintf(out + n, "%s\t%lld\t%lld", chrom, (long long)o.blk.v[3 * b], (long long)o.blk.v[3 * b + 1]);
        for (int64_t s = 0; s < S; s++) {
            const double m = orc_md_mean(depth + s * L, o.sites.v + s0, s1 - s0);
            int k = snprintf(tmp, sizeof tmp, "\t%.2f", m);
            memcpy(out + n, tmp, (size_t)k);
            n += (size_t)k;
        }
        out[n++] = '\n';
    }
    free(cls);
    free(o.blk.v);
    free(o.sites.v);
    *text = out;
    *len = (int64_t)n;
    return 0;
}

/* Batch of certification cells: cell i = depths d[off[i] .. off[i] + n[i]) over a span l[i].  out + i * stride gets the
 * NUL-terminated "%.2f" of the reference's chain. */
void orc_md_chain_batch(const int32_t* d, const int64_t* off, const int64_t* n, const int64_t* l, int64_t ncell, char* out, int stride) {
    for (int64_t i = 0; i < ncell; i++) {
        const double v = orc_md_chain(d + off[i], n[i], l[i]);
        snprintf(out + i * stride, (size_t)stride, "%.2f", v);
    }
}
