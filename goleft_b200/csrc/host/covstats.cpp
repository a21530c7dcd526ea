// covstats.cpp — see covstats.h; and the entries that need no device work of their own: gl_covstats_tail (arrays in, Stats
// out) and gl_bam_covstats_host (the host sampler + the same tail).
#include "covstats.h"
#include <math.h>
#include <string.h>
#include <chrono>
#include "bam_feed.h"

namespace glcs {

int SortedCounts::build(gl_ctx* ctx, const int32_t* v, size_t nv) {
    n = nv; cum.clear(); sorted.clear();
    if (nv == 0) return GL_OK;
    int32_t mn = v[0], mx = v[0];
    for (size_t i = 0; i < nv; i++) { mn = std::min(mn, v[i]); mx = std::max(mx, v[i]); }
    const long long range = (long long)mx - mn + 1;
    if (!ctx || range > kMaxHistRange || mx == INT32_MAX) { from_values(v, nv); return GL_OK; }
    std::vector<uint64_t> h((size_t)range, 0);
    const int rc = gl_bincount_i32(ctx, v, (int64_t)nv, mn, mx + 1, h.data());
    if (rc != GL_OK) return rc;
    from_hist(mn, std::move(h));
    return GL_OK;
}

void mean_std(const SortedCounts& a, size_t n, double& mean, double& sd) {
    const double l = (double)n;
    mean = 0; sd = 0;
    a.for_first(n, [&](int32_t x) { mean += (double)x / l; });
    const double mu = mean;
    a.for_first(n, [&](int32_t x) { sd += pow((double)x - mu, 2) / l; });
    sd = sqrt(sd);
}

size_t mad_filter(const SortedCounts& a, int nmads) {
    const size_t n = a.n;
    const int32_t med = a.kth(n / 2);
    // upper_mads = arr[n/2+1:] - med is already sorted: its middle element is arr[n/2+1 + len/2] - med
    const size_t len = n - (n / 2 + 1);
    const long long umad = (long long)a.kth(n / 2 + 1 + len / 2) - med;
    const long long upper = (long long)med + (long long)nmads * umad;
    size_t i = a.count_le(upper);                                                   // first index with arr[i] > upper
    if (i == n) i = n - 1;                                                          // Go's range loop leaves i at the last index
    return i;
}

int tail(gl_ctx* ctx, const SortedCounts& rl, const SortedCounts& ins, const SortedCounts& tm, gl_covstats* io, std::vector<double>& H) {
    H.clear();
    io->n_read_len = (int64_t)rl.n; io->n_insert = (int64_t)ins.n; io->h_len = 0;
    io->insert_mean = io->insert_sd = io->template_mean = io->template_sd = io->read_length_mean = io->read_length_median = 0;
    io->proportion_bad = io->proportion_unmapped = io->proportion_properly_paired = io->proportion_duplicate = 0;
    io->insert_pct5 = io->insert_pct95 = io->max_read_length = 0;
    if (rl.n > 0) {                                                                 // covstats.go:177-186
        const double den = (double)(io->k + io->n_unmapped);
        io->proportion_bad = (double)io->n_bad / den;
        io->proportion_duplicate = (double)io->n_dup / den;
        io->proportion_properly_paired = (double)io->n_proper / den;
        io->proportion_unmapped = (double)io->n_unmapped / den;
        io->read_length_median = (double)rl.kth((rl.n - 1) / 2) - 1;
        double sd;
        mean_std(rl, rl.n, io->read_length_mean, sd);
        io->max_read_length = rl.kth(rl.n - 1);
    }
    if (ins.n == 0) return GL_OK;
    const double l = (double)(ins.n - 1);                                           // covstats.go:188-199
    io->insert_pct5 = ins.kth((size_t)(0.05 * l + 0.5));
    io->insert_pct95 = ins.kth((size_t)(0.95 * l + 0.5));
    if (ins.n < 3 || tm.n < 3) return gl_fail(ctx, GL_EINVAL, "covstats: madFilter needs at least 3 insert sizes (the reference panics: index out of range)");
    mean_std(ins, mad_filter(ins, 10), io->insert_mean, io->insert_sd);
    const size_t kt = mad_filter(tm, 10);
    mean_std(tm, kt, io->template_mean, io->template_sd);
    const double start = (double)io->max_read_length;                              // covstats.go:202-217
    const double stop = io->template_mean + io->template_sd * 4;
    const double flen = stop - start + 1;
    if (!(flen > -1.0)) return gl_fail(ctx, GL_ERANGE, "covstats: the template histogram would have negative length (start %d, stop %g; the reference panics: makeslice: len out of range)", io->max_read_length, stop);
    if (flen >= 1e9) return gl_fail(ctx, GL_ERANGE, "covstats: the template histogram would have %g entries", flen);
    H.assign((size_t)(int64_t)flen, 0.0);
    double cnt = 0;
    tm.for_first(kt, [&](int32_t t) {
        const double x = (double)t;
        if (x < start || x > stop) return;
        H[(size_t)(int64_t)(x - start)] += 1;
        cnt += 1;
    });
    for (double& h : H) h /= cnt;                                                  // nothing in range: 0/0 = NaN, as in Go
    io->h_len = (int64_t)H.size();
    return GL_OK;
}

int put_hist(gl_ctx* ctx, const std::vector<double>& H, double* out, int64_t h_cap) {
    if ((int64_t)H.size() > h_cap || (!H.empty() && !out)) return gl_fail(ctx, GL_ERANGE, "covstats: H has %lld entries, room for %lld", (long long)H.size(), (long long)h_cap);
    if (!H.empty()) memcpy(out, H.data(), H.size() * sizeof(double));
    return GL_OK;
}

}  // namespace glcs

namespace {
double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
}

extern "C" {

int gl_covstats_tail(gl_ctx* ctx, const int32_t* read_len, int64_t n_read_len, const int32_t* insert, int64_t n_insert, const int32_t* tmpl,
                     int64_t n_tmpl, gl_covstats* io, double* H, int64_t h_cap) {
    if (!io || n_read_len < 0 || n_insert < 0 || n_tmpl < 0 || (n_read_len && !read_len) || (n_insert && !insert) || (n_tmpl && !tmpl))
        return gl_fail(ctx, GL_EINVAL, "gl_covstats_tail: bad argument");
    const double t0 = now_s();
    glcs::SortedCounts rl, ins, tm;
    int rc = rl.build(ctx, read_len, (size_t)n_read_len);
    if (rc == GL_OK) rc = ins.build(ctx, insert, (size_t)n_insert);
    if (rc == GL_OK) rc = tm.build(ctx, tmpl, (size_t)n_tmpl);
    if (rc != GL_OK) return rc;
    std::vector<double> h;
    rc = glcs::tail(ctx, rl, ins, tm, io, h);
    io->tail_s = now_s() - t0;
    if (rc != GL_OK) return rc;
    return glcs::put_hist(ctx, h, H, h_cap);
}

int gl_bam_covstats_host(gl_ctx* ctx, gl_bam* b, int32_t n, int32_t skip, gl_covstats* out, double* H, int64_t h_cap) {
    if (!b || !out) return gl_fail(ctx, GL_EINVAL, "gl_bam_covstats_host: null argument");
    memset(out, 0, sizeof *out);
    const double t0 = now_s();
    glhts::CovstatsSample cs;
    const std::string e = glhts::bam_covstats_sample(b->f, n, skip, cs);
    if (!e.empty()) return gl_fail(ctx, GL_EINVAL, "%s", e.c_str());
    out->n_unmapped = cs.n_unmapped; out->k = cs.k; out->n_bad = cs.n_bad; out->n_dup = cs.n_dup; out->n_proper = cs.n_proper;
    out->n_records_read = cs.n_read;
    out->read_s = now_s() - t0;                                                    // read + inflate + the record walk, interleaved
    const int rc = gl_covstats_tail(ctx, cs.read_len.data(), (int64_t)cs.read_len.size(), cs.insert.data(), (int64_t)cs.insert.size(),
                                    cs.tmpl.data(), (int64_t)cs.tmpl.size(), out, H, h_cap);
    b->cs = std::move(cs);
    out->wall_s = now_s() - t0;
    return rc;
}

int gl_bam_covstats_host_samples(gl_bam* b, const int32_t** read_len, const int32_t** insert, const int32_t** tmpl) {
    if (!b || !read_len || !insert || !tmpl) return GL_EINVAL;
    *read_len = b->cs.read_len.data(); *insert = b->cs.insert.data(); *tmpl = b->cs.tmpl.data();
    return GL_OK;
}

}  // extern "C"
