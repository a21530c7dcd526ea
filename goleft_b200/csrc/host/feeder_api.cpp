// feeder_api.cpp — C ABI over the host readers (hts_io): the segment feeder that replaces the
// `samtools depth` child's decode + filter (depth/depth.go:45) and biogo's BAI reader (indexcov.go:514), which
// here reads CSI too.
#include <string.h>
#include <string>
#include <vector>
#include "../../../include/goleft_b200.h"
#include "hts_io.h"
#include "bam_feed.h"

struct gl_segset { glhts::SegmentSet s; };
struct gl_bai { glhts::BaiIndex b; };

static void put_err(char* err, int64_t cap, const std::string& m) {
    if (!err || cap <= 0) return;
    const size_t n = m.size() < (size_t)cap - 1 ? m.size() : (size_t)cap - 1;
    memcpy(err, m.data(), n);
    err[n] = 0;
}

std::string gl_bam_plan_regions(gl_bam& b, int tid, const int64_t* beg, const int64_t* end, int64_t n,
                                std::vector<std::pair<uint64_t, uint64_t>>& out) {
    out.clear();
    if (!b.f.has_index) return "no index";
    if (!b.bins_read) {
        glhts::BaiIndex again;
        const std::string e = glhts::bai_read(b.f.index_path, again, &b.bins);
        if (!e.empty()) { b.bins.clear(); return e; }
        b.bins_read = true;
    }
    if (tid < 0 || tid >= (int)b.bins.size() || tid >= (int)b.f.bai.ioffsets.size()) return "";
    glhts::bai_region_chunks(b.bins[(size_t)tid], b.f.bai.ioffsets[(size_t)tid], b.f.bai.min_shift, b.f.bai.depth, beg, end, n, out);
    return "";
}

extern "C" {

int gl_bam_decode_segments(const char* path, int32_t min_mapq, int32_t threads, int32_t only_tid, gl_segset** out,
                           char* err, int64_t err_cap) {
    if (!path || !out) return GL_EINVAL;
    gl_segset* s = new gl_segset();
    const std::string e = glhts::bam_decode_segments(path, min_mapq, threads, only_tid, s->s);
    if (!e.empty()) { put_err(err, err_cap, e); delete s; *out = nullptr; return GL_EINVAL; }
    *out = s;
    return GL_OK;
}

int gl_segset_n_refs(const gl_segset* s, int32_t* n_refs, int64_t* n_records, int64_t* n_pass) {
    if (!s) return GL_EINVAL;
    if (n_refs) *n_refs = (int32_t)s->s.header.refs.size();
    if (n_records) *n_records = s->s.n_records;
    if (n_pass) *n_pass = s->s.n_pass;
    return GL_OK;
}

int gl_segset_ref(const gl_segset* s, int32_t tid, const char** name, int64_t* length, const int32_t** start,
                  const int32_t** end, int64_t* n) {
    if (!s || tid < 0 || tid >= (int32_t)s->s.header.refs.size()) return GL_EINVAL;
    if (name) *name = s->s.header.refs[tid].name.c_str();
    if (length) *length = s->s.header.refs[tid].length;
    if (start) *start = s->s.start[tid].data();
    if (end) *end = s->s.end[tid].data();
    if (n) *n = (int64_t)s->s.start[tid].size();
    return GL_OK;
}

void gl_segset_free(gl_segset* s) { delete s; }

int gl_bai_read(const char* path, gl_bai** out, char* err, int64_t err_cap) {
    if (!path || !out) return GL_EINVAL;
    gl_bai* b = new gl_bai();
    const std::string e = glhts::bai_read(path, b->b);
    if (!e.empty()) { put_err(err, err_cap, e); delete b; *out = nullptr; return GL_EINVAL; }
    *out = b;
    return GL_OK;
}

int gl_bai_n_refs(const gl_bai* b, int32_t* n_refs, uint64_t* n_no_coor) {
    if (!b) return GL_EINVAL;
    if (n_refs) *n_refs = (int32_t)b->b.ioffsets.size();
    if (n_no_coor) *n_no_coor = b->b.n_no_coor;
    return GL_OK;
}

int gl_bai_ref(const gl_bai* b, int32_t tid, const uint64_t** ioffsets, int64_t* n_intv, uint64_t* mapped, uint64_t* unmapped,
               int32_t* has_stats) {
    if (!b || tid < 0 || tid >= (int32_t)b->b.ioffsets.size()) return GL_EINVAL;
    if (ioffsets) *ioffsets = b->b.ioffsets[tid].data();
    if (n_intv) *n_intv = (int64_t)b->b.ioffsets[tid].size();
    if (mapped) *mapped = b->b.mapped[tid];
    if (unmapped) *unmapped = b->b.unmapped[tid];
    if (has_stats) *has_stats = b->b.has_stats[tid];
    return GL_OK;
}

int gl_bai_geometry(const gl_bai* b, int32_t* min_shift, int32_t* depth, int32_t* is_csi) {
    if (!b) return GL_EINVAL;
    if (min_shift) *min_shift = b->b.min_shift;
    if (depth) *depth = b->b.depth;
    if (is_csi) *is_csi = b->b.is_csi ? 1 : 0;
    return GL_OK;
}

void gl_bai_free(gl_bai* b) { delete b; }

// ---- index-guided parallel feeder (bam_feed.h)
int gl_bam_open(const char* path, gl_bam** out, char* err, int64_t err_cap) {
    if (!path || !out) return GL_EINVAL;
    gl_bam* b = new gl_bam();
    const std::string e = b->f.open(path);
    if (!e.empty()) { put_err(err, err_cap, e); delete b; *out = nullptr; return GL_EINVAL; }
    *out = b;
    return GL_OK;
}

void gl_bam_close(gl_bam* b) {
    if (b && b->cs_pf) cs_prefetch_drop(b->cs_pf);
    delete b;
}

int gl_bam_info(const gl_bam* b, int32_t* n_refs, int32_t* has_index) {
    if (!b) return GL_EINVAL;
    if (n_refs) *n_refs = (int32_t)b->f.header.refs.size();
    if (has_index) *has_index = b->f.has_index ? 1 : 0;
    return GL_OK;
}

int gl_bam_index(const gl_bam* b, const char** path, int32_t* min_shift, int32_t* depth, int32_t* is_csi) {
    if (!b) return GL_EINVAL;
    if (!b->f.has_index) return GL_ESTATE;
    if (path) *path = b->f.index_path.c_str();
    if (min_shift) *min_shift = b->f.bai.min_shift;
    if (depth) *depth = b->f.bai.depth;
    if (is_csi) *is_csi = b->f.bai.is_csi ? 1 : 0;
    return GL_OK;
}

int gl_bam_ref(const gl_bam* b, int32_t tid, const char** name, int64_t* length, int64_t* n_mapped) {
    if (!b || tid < 0 || tid >= (int32_t)b->f.header.refs.size()) return GL_EINVAL;
    if (name) *name = b->f.header.refs[tid].name.c_str();
    if (length) *length = b->f.header.refs[tid].length;
    if (n_mapped) *n_mapped = (b->f.has_index && tid < (int32_t)b->f.bai.mapped.size() && b->f.bai.has_stats[tid]) ? (int64_t)b->f.bai.mapped[tid] : -1;
    return GL_OK;
}

int gl_bam_decode(gl_bam* b, int32_t tid, int64_t beg, int64_t end, int32_t min_mapq, int32_t threads, int32_t want_format,
                  gl_bam_segments* out, char* err, int64_t err_cap) {
    if (!b || !out) return GL_EINVAL;
    memset(out, 0, sizeof *out);
    glhts::DecodeStats st;
    const std::string e = b->f.decode(tid, beg, end, min_mapq, threads, want_format, b->segs, &st);
    if (!e.empty()) { put_err(err, err_cap, e); return GL_EINVAL; }
    out->format = b->segs.format;
    if (b->segs.format == 8) {
        out->n = b->segs.n_blocks; out->a0 = b->segs.anchors.data(); out->a1 = b->segs.ds.data(); out->a2 = b->segs.len.data();
    } else if (b->segs.format == 32) {
        out->n = b->segs.n; out->a0 = b->segs.start.data(); out->a1 = b->segs.end.data(); out->a2 = nullptr;
    }
    out->n_records = st.n_records; out->n_pass = st.n_pass; out->bytes_in = st.bytes_in; out->bytes_out = st.bytes_out;
    out->inflate_s = st.inflate_s; out->parse_s = st.parse_s; out->wall_s = st.wall_s; out->units = st.units;
    out->max_len = b->segs.max_len;
    return GL_OK;
}

int gl_bam_region_chunks(const gl_bam* b, int32_t tid, const int64_t* beg, const int64_t* end, int64_t n, uint64_t* vb, uint64_t* ve,
                         int64_t cap, int64_t* n_out) {
    if (!b || !n_out || n < 0 || (n > 0 && (!beg || !end)) || cap < 0 || (cap > 0 && (!vb || !ve))) return GL_EINVAL;
    *n_out = 0;
    if (!b->f.has_index) return GL_ESTATE;
    if (tid < 0 || tid >= (int32_t)b->f.header.refs.size()) return GL_EINVAL;
    std::vector<std::pair<uint64_t, uint64_t>> r;
    if (!gl_bam_plan_regions(const_cast<gl_bam&>(*b), tid, beg, end, n, r).empty()) return GL_ESTATE;   // fills the handle's bin cache
    *n_out = (int64_t)r.size();
    if ((int64_t)r.size() > cap) return GL_ERANGE;
    for (size_t i = 0; i < r.size(); i++) { vb[i] = r[i].first; ve[i] = r[i].second; }
    return GL_OK;
}

int gl_crai_make_sizes(const int64_t* aln_start, const int64_t* aln_span, const int32_t* slice_len, int64_t n, int64_t* sizes,
                       int64_t cap, int64_t* n_sizes) {
    if (n < 0 || !n_sizes || (n > 0 && (!aln_start || !aln_span || !slice_len))) return GL_EINVAL;
    std::vector<int64_t> v;
    if (!glhts::crai_make_sizes(aln_start, aln_span, slice_len, n, v)) return GL_ERANGE;    // the reference panics here
    *n_sizes = (int64_t)v.size();
    if ((int64_t)v.size() > cap) return GL_ERANGE;
    if (!v.empty()) memcpy(sizes, v.data(), v.size() * sizeof(int64_t));
    return GL_OK;
}

}  // extern "C"
