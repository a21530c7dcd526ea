// bam_feed.cpp — see bam_feed.h.  BGZF / BAM / BAI layouts: SAM spec sections 4.1, 4.2, 5.2 (SURVEY.md Appendix D).
#include "bam_feed.h"
#include <fcntl.h>
#include <string.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <mutex>
#include "bam_cigar.h"
#include "seg_pack.h"
#include "thread_pool.h"

namespace glhts {

using glhost::Piece;

namespace {

inline uint16_t rd16(const uint8_t* p) { return (uint16_t)(p[0] | (p[1] << 8)); }
inline uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
inline int32_t rdi32(const uint8_t* p) { return (int32_t)rd32(p); }

constexpr int64_t kUnitBytes = 1 << 20;          // compressed bytes per work unit (about 64 tiles of a 30x BAM)
constexpr int64_t kWindow = (1 << 20) + (1 << 16);
constexpr int64_t kStreamChunk = int64_t(32) << 20;   // compressed bytes per BamFile::stream read

// size of the BGZF block at p (0: not a block header / not enough bytes to tell)
size_t block_size(const uint8_t* p, size_t avail) {
    if (avail < 18) return 0;
    if (p[0] != 0x1f || p[1] != 0x8b || p[2] != 8 || !(p[3] & 4)) return 0;
    const uint16_t xlen = rd16(p + 10);
    size_t q = 12;
    while (q + 4 <= 12u + xlen && q + 4 <= avail) {
        const uint16_t slen = rd16(p + q + 2);
        if (p[q] == 'B' && p[q + 1] == 'C' && slen == 2 && q + 6 <= avail) return (size_t)rd16(p + q + 4) + 1;
        q += 4u + slen;
    }
    return 0;
}

struct Inflater {                                 // one z_stream per thread (inflater()), reset per block
    z_stream zs;
    bool ok = false;
    Inflater() { memset(&zs, 0, sizeof zs); ok = inflateInit2(&zs, -15) == Z_OK; }
    ~Inflater() { if (ok) inflateEnd(&zs); }
    bool block(const uint8_t* src, size_t csize, uint8_t* dst, uint32_t isize) {
        const uint16_t xlen = rd16(src + 10);
        const size_t hdr = 12u + xlen;
        if (csize < hdr + 8) return false;
        if (isize == 0) return true;
        if (!ok || inflateReset(&zs) != Z_OK) return false;
        zs.next_in = const_cast<Bytef*>(src + hdr);
        zs.avail_in = (uInt)(csize - hdr - 8);
        zs.next_out = dst;
        zs.avail_out = isize;
        const int rc = inflate(&zs, Z_FINISH);
        return rc == Z_STREAM_END && zs.total_out == isize;
    }
};

Inflater& inflater() {
    thread_local Inflater inf;
    return inf;
}

struct Unit { uint64_t v0 = 0, v1 = 0; };

struct UnitOut {
    std::vector<Piece> list;                      // (start, length), sorted by start
    int64_t n_records = 0, n_pass = 0, bytes_in = 0, bytes_out = 0, sum_len = 0;
    int32_t max_len = 0;
    double inflate_s = 0, parse_s = 0;
    std::string err;
};

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// the M/=/X blocks of one record into `pend` (kept sorted by start), after moving everything that starts at or
// before this record's position to `out`: later records start at or after it, so `out` stays sorted
struct Emitter {
    std::vector<Piece>& out;
    std::vector<Piece> pend;
    int32_t last_pos = INT32_MIN;
    bool sorted = true;
    int64_t sum_len = 0;
    int32_t max_len = 0;
    explicit Emitter(std::vector<Piece>& o) : out(o) {}
    inline void flush_upto(int32_t pos) {
        size_t k = 0;
        while (k < pend.size() && pend[k].first <= pos) out.push_back(pend[k++]);
        if (k) pend.erase(pend.begin(), pend.begin() + (long)k);
    }
    inline void add(int32_t s, int32_t len) {
        sum_len += len;
        if (len > max_len) max_len = len;
        size_t j = pend.size();
        pend.emplace_back(s, len);
        while (j > 0 && pend[j - 1].first > s) { pend[j] = pend[j - 1]; j--; }
        pend[j] = Piece(s, len);
    }
    inline void record(const uint8_t* r, uint32_t bs) {
        const int32_t pos = rdi32(r + 4);
        if (pos < last_pos) sorted = false;         // not coordinate-sorted: fixed up at the end
        last_pos = pos;
        if (!pend.empty()) flush_upto(pos);
        glbam::depth_blocks(r, bs, [&](int32_t b, int32_t e) { add(b, e - b); });
    }
    void finish() {
        for (const Piece& p : pend) out.push_back(p);
        pend.clear();
        if (!sorted) glhost::sort_nearly_sorted(out.data(), out.size());
    }
};

}  // namespace

BamFile::~BamFile() { if (fd_ >= 0) close(fd_); }

std::string BamFile::open(const std::string& p, bool with_index) {
    path = p;
    fd_ = ::open(p.c_str(), O_RDONLY);
    if (fd_ < 0) return "cannot open " + p;
    struct stat st;
    if (fstat(fd_, &st) != 0) return "cannot stat " + p;
    size_ = (int64_t)st.st_size;
    // header: inflate block by block until it parses (a header is a few blocks; the old reader inflated 32 MB)
    std::vector<uint8_t> cin, text;
    Inflater& inf = inflater();
    int64_t c = 0;
    bool done = false;
    while (!done && c < size_) {
        const int64_t want = std::min<int64_t>(1 << 18, size_ - c);
        cin.resize((size_t)want);
        const ssize_t got = pread(fd_, cin.data(), (size_t)want, c);
        if (got <= 0) break;
        size_t q = 0;
        bool any = false;
        while (q < (size_t)got) {
            const size_t bs = block_size(cin.data() + q, (size_t)got - q);
            if (bs == 0 || q + bs > (size_t)got) break;
            const uint32_t isize = rd32(cin.data() + q + bs - 4);
            if (isize > 65536) return "bad BGZF ISIZE in " + p;
            const size_t at = text.size();
            text.resize(at + isize);
            if (!inf.block(cin.data() + q, bs, text.data() + at, isize)) return "inflate failed in " + p;
            q += bs;
            any = true;
            // try to parse
            if (text.size() >= 12) {
                if (memcmp(text.data(), "BAM\1", 4) != 0) return "not a BAM file: " + p;
                const uint32_t l_text = rd32(text.data() + 4);
                if (text.size() >= 8 + (size_t)l_text + 4) {
                    const uint32_t n_ref = rd32(text.data() + 8 + l_text);
                    size_t o = 8 + (size_t)l_text + 4;
                    std::vector<RefInfo> refs;
                    bool complete = true;
                    for (uint32_t r = 0; r < n_ref; r++) {
                        if (text.size() < o + 4) { complete = false; break; }
                        const uint32_t l_name = rd32(text.data() + o);
                        if (text.size() < o + 4 + l_name + 4) { complete = false; break; }
                        RefInfo ri;
                        ri.name.assign(reinterpret_cast<const char*>(text.data() + o + 4), l_name ? l_name - 1 : 0);
                        ri.length = rdi32(text.data() + o + 4 + l_name);
                        refs.push_back(ri);
                        o += 4 + l_name + 4;
                    }
                    if (complete) {
                        header.text.assign(reinterpret_cast<const char*>(text.data() + 8), l_text);
                        while (!header.text.empty() && header.text.back() == 0) header.text.pop_back();
                        header.refs = refs;
                        rec_member_ = c + (int64_t)(q - bs);            // the header ends in this member
                        rec_skip_ = (uint32_t)(o - at);
                        done = true;
                        break;
                    }
                }
            }
        }
        if (!any) break;
        c += (int64_t)q;
    }
    if (!done) return "truncated BAM header: " + p;
    if (!with_index) return "";
    for (const std::string& ip : index_candidates(p)) {
        struct stat s2;
        if (stat(ip.c_str(), &s2) != 0) continue;
        BaiIndex b;
        if (bai_read(ip, b).empty()) { bai = std::move(b); has_index = true; index_path = ip; break; }
    }
    return "";
}

std::string BamFile::decode(int tid, int64_t beg, int64_t end, int min_mapq, int threads, int want, ContigSegs& out, DecodeStats* st) {
    const double t_wall = now_s();
    out = ContigSegs();
    if (fd_ < 0) return "BAM not open";
    if (!has_index) return "no .bai or .csi index for " + path;
    if (tid < 0 || tid >= (int)header.refs.size() || tid >= (int)bai.ioffsets.size()) return "";
    const std::vector<uint64_t>& lin = bai.ioffsets[(size_t)tid];
    const int64_t ref_len = header.refs[(size_t)tid].length;
    if (beg < 0) beg = 0;
    if (end > ref_len) end = ref_len;
    if (lin.empty() || end <= beg) return "";
    // past a BAI's linear index no record reaches the region; a CSI's rebuilt one ends at the last tile a bin starts in, and
    // a record that starts before it may reach further: start from its last entry
    const int64_t t0 = bai.is_csi ? std::min<int64_t>(beg >> 14, (int64_t)lin.size() - 1) : beg >> 14;
    if (t0 >= (int64_t)lin.size()) return "";                        // no record reaches the region
    const int64_t t1 = std::min<int64_t>((int64_t)lin.size() - 1, (end - 1) >> 14);
    // ---- units: cut at linear-index offsets (each is the first record overlapping a 16 KB tile: record-aligned)
    std::vector<Unit> units;
    uint64_t cur = 0;
    for (int64_t t = t0; t <= t1; t++) {
        const uint64_t v = lin[(size_t)t];
        if (v == 0) continue;
        if (cur == 0) { cur = v; units.push_back(Unit{v, 0}); continue; }
        if (v > units.back().v0 && (int64_t)(v >> 16) - (int64_t)(units.back().v0 >> 16) >= kUnitBytes) units.push_back(Unit{v, 0});
    }
    if (units.empty()) return "";
    // end of the stream: the reference's last record (max chunk end over its bins) — a query that stops inside the
    // reference also stops at the first record at or beyond `end` (records are sorted), whichever comes first
    uint64_t vend = tid < (int)bai.ref_end.size() ? bai.ref_end[(size_t)tid] : 0;
    if (vend == 0) {
        for (size_t r = (size_t)tid + 1; r < bai.ref_beg.size() && vend == 0; r++) vend = bai.ref_beg[r];
        if (vend == 0) vend = (uint64_t)size_ << 16;
    }
    for (size_t u = 0; u + 1 < units.size(); u++) units[u].v1 = units[u + 1].v0;
    units.back().v1 = std::max(vend, units.back().v0);
    const int64_t end_pos = end;

    std::vector<UnitOut> res(units.size());
    glhost::ThreadPool& pool = glhost::ThreadPool::global();
    const int T = threads > 0 ? std::min(threads, pool.size()) : pool.size();
    pool.run((int64_t)units.size(), [&](int64_t ui, int) {
        UnitOut& R = res[(size_t)ui];
        const Unit& U = units[(size_t)ui];
        thread_local std::vector<uint8_t> cin, buf;
        Inflater& inf = inflater();
        cin.resize((size_t)kWindow);
        buf.clear();
        size_t pos = 0;
        Emitter em(R.list);
        R.list.reserve(1 << 16);
        int64_t c = (int64_t)(U.v0 >> 16);
        size_t skip = (size_t)(U.v0 & 0xffff);
        const int64_t cend = (int64_t)(U.v1 >> 16);
        const uint32_t uend = (uint32_t)(U.v1 & 0xffff);
        bool done_reading = false, finished = false;
        while (!finished) {
            if (!done_reading) {
                const int64_t want = std::min<int64_t>(kWindow, size_ - c);
                if (want <= 0) done_reading = true;
                else {
                    const double ti = now_s();
                    const ssize_t got = pread(fd_, cin.data(), (size_t)want, c);
                    if (got <= 0) { R.err = "read failed in " + path; return; }
                    size_t q = 0;
                    bool any = false;
                    while (q < (size_t)got) {
                        const int64_t cb = c + (int64_t)q;
                        if (cb > cend || (cb == cend && uend == 0)) { done_reading = true; break; }
                        const size_t bs = block_size(cin.data() + q, (size_t)got - q);
                        if (bs == 0) {
                            if ((size_t)got - q >= 18) { R.err = "not a BGZF block in " + path; return; }
                            break;
                        }
                        if (q + bs > (size_t)got) break;
                        const uint32_t isize = rd32(cin.data() + q + bs - 4);
                        if (isize > 65536) { R.err = "bad BGZF ISIZE in " + path; return; }
                        const size_t at = buf.size();
                        buf.resize(at + isize);
                        if (!inf.block(cin.data() + q, bs, buf.data() + at, isize)) { R.err = "inflate failed in " + path; return; }
                        R.bytes_in += (int64_t)bs;
                        R.bytes_out += isize;
                        if (cb == cend) { buf.resize(at + std::min<uint32_t>(uend, isize)); done_reading = true; }
                        if (skip) {                                           // the unit starts inside its first block
                            const size_t k = std::min(skip, buf.size() - at);
                            buf.erase(buf.begin() + (long)at, buf.begin() + (long)(at + k));
                            skip = 0;
                        }
                        q += bs;
                        any = true;
                        if (done_reading) break;
                    }
                    c += (int64_t)q;
                    if (!any && !done_reading) {
                        if (c + (int64_t)got >= size_) done_reading = true;     // trailing bytes that are not a whole block
                        else { R.err = "truncated BGZF block in " + path; return; }
                    }
                    R.inflate_s += now_s() - ti;
                }
            }
            // ---- records
            const double tp = now_s();
            for (;;) {
                const size_t av = buf.size() - pos;
                if (av < 4) break;
                const uint32_t bs = rd32(buf.data() + pos);
                if (bs < 32) { R.err = "corrupt BAM record in " + path; return; }
                if (av < 4 + (size_t)bs) break;
                const uint8_t* r = buf.data() + pos + 4;
                pos += 4 + bs;
                const int32_t rtid = rdi32(r), rpos = rdi32(r + 4);
                if (rtid != tid) { if (rtid > tid || rtid < 0) { finished = true; break; } continue; }
                if (rpos >= end_pos) { finished = true; break; }
                R.n_records++;
                if (!glbam::depth_counts(r, bs, min_mapq)) continue;
                R.n_pass++;
                em.record(r, bs);
            }
            R.parse_s += now_s() - tp;
            if (done_reading) break;
            if (pos > (size_t(4) << 20)) { buf.erase(buf.begin(), buf.begin() + (long)pos); pos = 0; }
        }
        em.finish();
        R.sum_len = em.sum_len;
        R.max_len = em.max_len;
        if (buf.capacity() > (size_t(64) << 20)) { std::vector<uint8_t>().swap(buf); }
    }, T);
    DecodeStats S;
    S.units = (int)units.size();
    int64_t sum_len = 0;
    for (UnitOut& R : res) {
        if (!R.err.empty()) return R.err;
        S.n_records += R.n_records; S.n_pass += R.n_pass; S.bytes_in += R.bytes_in; S.bytes_out += R.bytes_out;
        S.inflate_s += R.inflate_s; S.parse_s += R.parse_s;
        out.n_pieces += (int64_t)R.list.size();
        out.max_len = std::max(out.max_len, R.max_len);
        sum_len += R.sum_len;
    }
    if (out.n_pieces > 0) {
        // packed8 pays for short blocks only: a 10 kb block would become 40 pieces of 2 bytes against 8 bytes as int32
        int fmt = want;
        if (fmt != 8 && fmt != 32) fmt = (sum_len <= 400 * out.n_pieces) ? 8 : 32;
        std::vector<const std::vector<Piece>*> lists(res.size());
        if (fmt == 8 && out.max_len > 255)
            pool.run((int64_t)res.size(), [&](int64_t k, int) { glhost::split_long_pieces(res[(size_t)k].list); }, T);
        for (size_t k = 0; k < res.size(); k++) lists[k] = &res[k].list;
        glhost::Assembled A;
        if (fmt == 8) {
            glhost::assemble_p8(lists, T, A);
            out.n_blocks = A.total;
            out.anchors.resize((size_t)A.total);
            out.ds.resize((size_t)A.total * 64);
            out.len.resize((size_t)A.total * 64);
            glhost::concat_p8(A, T, out.anchors.data(), out.ds.data(), out.len.data());
        } else {
            glhost::assemble_i32(lists, T, A);
            out.n = A.total;
            out.start.resize((size_t)A.total);
            out.end.resize((size_t)A.total);
            glhost::concat_i32(A, T, out.start.data(), out.end.data());
        }
        out.format = fmt;
    }
    S.wall_s = now_s() - t_wall;
    if (st) *st = S;
    return "";
}

std::string BamFile::stream(int threads, const std::function<bool(const uint8_t*, uint32_t)>& fn) {
    if (fd_ < 0) return "BAM not open";
    glhost::ThreadPool& pool = glhost::ThreadPool::global();
    const int T = threads > 0 ? std::min(threads, pool.size()) : pool.size();
    struct Member { size_t at, size, out; uint32_t isize; };
    std::vector<Member> mem;
    std::vector<uint8_t> cin, buf;                    // buf: the record cut by the last chunk's end, then this chunk inflated
    size_t carry = 0, pos = rec_skip_;
    int64_t c = rec_member_;
    while (c < size_) {
        const size_t want = (size_t)std::min<int64_t>(kStreamChunk, size_ - c);
        cin.resize(want);
        for (size_t got = 0; got < want;) {
            const ssize_t k = pread(fd_, cin.data() + got, want - got, c + (int64_t)got);
            if (k <= 0) return "read failed in " + path;
            got += (size_t)k;
        }
        const bool eof = c + (int64_t)want == size_;
        // the chunk's whole members; the one its end cuts is read again with the next chunk
        mem.clear();
        size_t q = 0, out = carry;
        while (q < want) {
            const size_t bs = block_size(cin.data() + q, want - q);
            if (bs == 0) {
                if (!eof && want - q < 18) break;
                return "not a BGZF block in " + path;
            }
            if (q + bs > want) {
                if (eof) return "truncated BGZF block in " + path;
                break;
            }
            const uint32_t isize = rd32(cin.data() + q + bs - 4);
            if (isize > 65536) return "bad BGZF ISIZE in " + path;
            mem.push_back(Member{q, bs, out, isize});
            out += isize;
            q += bs;
        }
        c += (int64_t)q;
        buf.resize(out);
        std::atomic<bool> bad(false);
        pool.run((int64_t)mem.size(), [&](int64_t i, int) {
            const Member& m = mem[(size_t)i];
            if (!inflater().block(cin.data() + m.at, m.size, buf.data() + m.out, m.isize)) bad = true;
        }, T);
        if (bad) return "inflate failed in " + path;
        for (;;) {
            const size_t av = buf.size() - pos;
            if (av < 4) break;
            const uint32_t bs = rd32(buf.data() + pos);
            if (bs < 32) return "corrupt BAM record: " + path;
            if (av < 4 + (size_t)bs) break;
            if (!fn(buf.data() + pos + 4, bs)) return "";
            pos += 4 + (size_t)bs;
        }
        carry = buf.size() - pos;
        memmove(buf.data(), buf.data() + pos, carry);
        pos = 0;
    }
    return "";
}

std::string bam_read_header(const std::string& path, BamHeader& out) {
    BamFile f;
    const std::string err = f.open(path, false);
    if (!err.empty()) return err;
    out = f.header;
    return "";
}

std::string bam_decode_segments(const std::string& path, int min_mapq, int threads, int only_tid, SegmentSet& out) {
    BamFile f;
    const std::string err = f.open(path, false);
    if (!err.empty()) return err;
    out.header = f.header;
    const int32_t n_ref = (int32_t)out.header.refs.size();
    out.start.assign((size_t)n_ref, {});
    out.end.assign((size_t)n_ref, {});
    out.n_records = out.n_pass = 0;
    return f.stream(std::max(threads, 1), [&](const uint8_t* r, uint32_t bs) {
        out.n_records++;
        const int32_t tid = rdi32(r);
        if (tid < 0 || tid >= n_ref || (only_tid >= 0 && tid != only_tid)) return true;
        if (!glbam::depth_counts(r, bs, min_mapq)) return true;
        out.n_pass++;
        std::vector<int32_t>& S = out.start[(size_t)tid];
        std::vector<int32_t>& E = out.end[(size_t)tid];
        glbam::depth_blocks(r, bs, [&](int32_t b, int32_t e) { S.push_back(b); E.push_back(e); });
        return true;
    });
}

// covstats reads the stored CIGAR: the reference reads BAM through biogo/hts, whose handling of CG is not established
std::string bam_covstats_sample(BamFile& f, int n, int skip, CovstatsSample& o) {
    o = CovstatsSample();
    if (n <= 0) return "";                                                     // :138 is false at once: nothing is sampled
    int64_t seen = 0;
    return f.stream(0, [&](const uint8_t* r, uint32_t size) {
        if (seen++ < skip) { o.n_read = seen; return true; }                   // covstats.go:128-134
        if ((int64_t)o.insert.size() >= n) return false;                       // :138
        o.n_read = seen;
        const int32_t pos = rdi32(r + 4);
        const uint8_t l_name = r[8];
        const uint16_t n_cig = rd16(r + 12), flag = rd16(r + 14);
        const int32_t mate_pos = rdi32(r + 24), tlen = rdi32(r + 28);
        if (flag & 0x4) { o.n_unmapped++; return true; }                       // :144-147
        o.k++;
        if (flag & (0x400 | 0x200)) {                                          // :149-155
            if (flag & 0x400) o.n_dup++;
            o.n_bad++;
            return true;
        }
        if (flag & 0x2) o.n_proper++;                                          // :156-158
        if (32u + l_name + 4u * n_cig > size) return true;
        const uint8_t* cg = r + 32 + l_name;
        int32_t ref_len = 0, read_len = 0;
        for (uint16_t k = 0; k < n_cig; k++) {
            const uint32_t v = rd32(cg + 4 * k), op = v & 15, len = v >> 4;
            if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) ref_len += (int32_t)len;
            if (op == 0 || op == 1 || op == 4 || op == 7 || op == 8) read_len += (int32_t)len;
        }
        if ((int64_t)o.read_len.size() < 2 * (int64_t)n) o.read_len.push_back(read_len);      // :159-161
        else if (o.insert.empty()) return false;                                               // :163-166
        if (pos < mate_pos && (flag & 0x2) && n_cig == 1 && (rd32(cg) & 15) == 0) {            // :169-172
            o.insert.push_back(mate_pos - (pos + ref_len));
            o.tmpl.push_back(tlen);
        }
        return true;
    });
}

}  // namespace glhts
