// multidepth.cpp — host side of `goleft multidepth` (multidepth/multidepth.go): the chunk state machine that turns the
// contig's site classes into blocks, the certification of a mean's digits, and the row text.
//
// The reference walks `samtools depth` lines one site at a time (aggregate, :202-266).  Here the same decisions are taken
// per run of one site class (absent / insufficient / sufficient, from gl_multidepth_sites): inside an insufficient run the
// cache does not change, so the first site where the chain breaks or the chunk is killed follows from arithmetic; a
// sufficient run joins the chain (or replaces it) as a whole.  The cache is kept as a list of sufficient runs.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <string>
#include <vector>
#include "../../../include/goleft_b200.h"
#include "md_cert.h"
#include "thread_pool.h"

namespace {

struct Run { int64_t a, b; };                          // [a, b): consecutive sufficient sites

struct Blocks {
    std::vector<int64_t> s, e, n;
    int64_t window;
    // splitBlocks (:183-200) over a cache of runs: a block starts at a cached site and takes the cached sites < start + Window
    void split(const std::vector<Run>& cache) {
        const int64_t w = std::max<int64_t>(window, 1);    // Window <= 1: every site is its own block, as in the reference
        size_t i = 0;
        int64_t p = cache.empty() ? 0 : cache[0].a;
        while (i < cache.size()) {
            const int64_t start = p, limit = start + w;
            int64_t cnt = 0, last = start;
            while (i < cache.size()) {
                const int64_t a = std::max(cache[i].a, p), b = cache[i].b;
                if (a >= limit) { p = a; break; }
                const int64_t e = std::min(b, limit);
                cnt += e - a;
                last = e - 1;
                if (e < b) { p = e; break; }
                i++;
                if (i < cache.size()) p = cache[i].a;
            }
            s.push_back(start);
            e.push_back(last + 1);
            n.push_back(cnt);
        }
    }
};

struct Chain {
    std::vector<Run> cache;
    int64_t sites = 0;
    int64_t last() const { return cache.back().b - 1; }
    bool empty() const { return cache.empty(); }
    void clear() { cache.clear(); sites = 0; }
    void append(int64_t a, int64_t b) {
        if (!cache.empty() && cache.back().b == a) cache.back().b = b;
        else cache.push_back({a, b});
        sites += b - a;
    }
};

}  // namespace

extern "C" {

int gl_multidepth_blocks(const int32_t* run_start, const uint8_t* run_class, int64_t n_runs, int64_t contig_len, int32_t n_samples,
                         int64_t chunk, int64_t max_skip, int64_t min_size, int64_t window, int64_t* blk_start, int64_t* blk_end,
                         int64_t* blk_sites, int64_t cap, int64_t* n_blocks) {
    if (n_runs < 0 || contig_len < 0 || (n_runs > 0 && (!run_start || !run_class)) || !n_blocks || n_samples < 1 || chunk < 0)
        return GL_EINVAL;
    for (int64_t i = 0; i < n_runs; i++)
        if (run_class[i] > 2 || run_start[i] < 0 || run_start[i] >= contig_len || (i > 0 && run_start[i] <= run_start[i - 1]))
            return GL_EINVAL;
    const int64_t C = chunk > 0 ? chunk : (n_samples > 50 ? 5000000 / 5 : 5000000);   // multidepth.go:60-62,121
    Blocks out;
    out.window = window;
    Chain ch;
    for (int64_t k0 = 0; k0 < contig_len; k0 += C) {
        const int64_t T = k0 + 1 + C;                 // kill sites lie beyond r.start + chunkSize (r.start is 1-based)
        ch.clear();
        bool seen0 = false, killed = false;
        // first run that reaches k0
        int64_t i = std::upper_bound(run_start, run_start + n_runs, (int32_t)std::min<int64_t>(k0, INT32_MAX)) - run_start - 1;
        if (i < 0) i = 0;
        for (; i < n_runs && !killed; i++) {
            const int64_t a = std::max<int64_t>(run_start[i], k0);
            const int64_t b = i + 1 < n_runs ? run_start[i + 1] : contig_len;
            if (a >= b || run_class[i] == 0) continue;
            if (run_class[i] == 1) {
                seen0 = true;
                int64_t from = a;                       // the next site of this run to look at
                if (!ch.empty()) {
                    const int64_t last = ch.last();
                    const int64_t kill_at = std::max(T + 1, last + max_skip);      // first site that kills with this cache
                    const int64_t brk_at = last + max_skip + 2;                     // first site that breaks the chain
                    const int64_t ev = std::max(a, std::min(kill_at, brk_at));
                    if (ev >= b) continue;
                    if (ev > T && ev - last >= max_skip) { killed = true; break; }
                    // the chain breaks at ev (MinSize applies), the cache is empty from here on
                    if (ch.sites >= min_size) out.split(ch.cache);
                    ch.clear();
                    from = ev + 1;
                }
                const int64_t kill_at = std::max(from, T + 1);                     // empty cache: any site beyond T kills
                if (kill_at < b) { killed = true; break; }
            } else {
                if (!seen0) continue;
                if (!ch.empty() && a - (ch.last() + 1) > max_skip) {
                    if (ch.sites >= min_size) out.split(ch.cache);
                    ch.clear();
                }
                ch.append(a, b);
            }
        }
        if (!ch.empty()) out.split(ch.cache);     // the cache left at the kill / contig end: no MinSize test (:259-263)
    }
    const int64_t nb = (int64_t)out.s.size();
    *n_blocks = nb;
    if (!blk_start && !blk_end && !blk_sites) return GL_OK;
    if (nb > cap || !blk_start || !blk_end || !blk_sites) return GL_ERANGE;
    for (int64_t k = 0; k < nb; k++) { blk_start[k] = out.s[k]; blk_end[k] = out.e[k]; blk_sites[k] = out.n[k]; }
    return GL_OK;
}

int gl_multidepth_certify(const int64_t* sum, const int64_t* n_sites, const int64_t* span, int64_t n, int64_t* q, uint8_t* certified) {
    if (n < 0 || (n > 0 && (!sum || !n_sites || !span || !q || !certified))) return GL_EINVAL;
    for (int64_t i = 0; i < n; i++) {
        int64_t v = 0;
        certified[i] = glmd::certify((uint64_t)sum[i], n_sites[i], span[i], &v) ? 1 : 0;
        q[i] = certified[i] ? v : 0;
    }
    return GL_OK;
}

int gl_multidepth_text(const char* chrom, const int64_t* blk_start, const int64_t* blk_end, int64_t n_blocks, int32_t S, const int64_t* q,
                       const double* val, const uint8_t* certified, int32_t threads, char** text, int64_t* text_len) {
    if (!chrom || !text || !text_len || S < 1 || n_blocks < 0 || (n_blocks > 0 && (!blk_start || !blk_end || !q || !val || !certified)))
        return GL_EINVAL;
    // rows are independent: groups of rows are formatted on the host pool and concatenated in order
    const int64_t per = 4096;
    const int64_t groups = (n_blocks + per - 1) / per;
    std::vector<std::string> parts((size_t)groups);
    auto fmt = [&](int64_t g, int) {
        std::string& o = parts[(size_t)g];
        char buf[64];
        for (int64_t b = g * per; b < std::min(n_blocks, (g + 1) * per); b++) {
            o += chrom;
            snprintf(buf, sizeof buf, "\t%lld\t%lld", (long long)blk_start[b], (long long)blk_end[b]);
            o += buf;
            for (int32_t s = 0; s < S; s++) {
                const size_t c = (size_t)b * S + s;
                if (certified[c]) snprintf(buf, sizeof buf, "\t%lld.%02lld", (long long)(q[c] / 100), (long long)(q[c] % 100));
                else snprintf(buf, sizeof buf, "\t%.2f", val[c]);
                o += buf;
            }
            o += '\n';
        }
    };
    if (groups > 1) glhost::ThreadPool::global().run(groups, fmt, threads);
    else if (groups == 1) fmt(0, 0);
    size_t total = 0;
    for (const std::string& p : parts) total += p.size();
    char* out = (char*)malloc(total + 1);
    if (!out) return GL_ENOMEM;
    size_t off = 0;
    for (const std::string& p : parts) { memcpy(out + off, p.data(), p.size()); off += p.size(); }
    out[total] = 0;
    *text = out;
    *text_len = (int64_t)total;
    return GL_OK;
}

}  // extern "C"
