// goleft — C++ host for the H100 engine, keeping the `goleft depth|indexcov|covstats|depthwed` command-line
// and BED/TSV output surface of brentp/goleft v0.2.6 (cmd/goleft/goleft.go:24-69).  Every number it prints is
// computed by libgoleft_b200.so (CUDA, sm_90a) through the C ABI in include/goleft_b200.h; there is no CPU
// fallback: without a GPU the subcommands fail with the library's error.
//
// Out of scope here (SURVEY.md §2): HTML/PNG plots, --stats GC columns.  .crai input needs --fai.
#include <errno.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <time.h>
#include <unistd.h>
#include <algorithm>
#include <array>
#include <chrono>
#include <functional>
#include <condition_variable>
#include <map>
#include <mutex>
#include <regex>
#include <set>
#include <string>
#include <thread>
#include <vector>
#include <zlib.h>

#include "../goleft_b200/csrc/host/hts_io.h"
#include "../goleft_b200/csrc/host/bam_feed.h"
#include "../goleft_b200/csrc/host/thread_pool.h"
#include "../goleft_b200/csrc/host/pca8.h"
#include "goleft_b200.h"
#include "plot_html.h"

static const char* kVersion = "0.2.6";          // goleft.go:3 (the surface this build mirrors)

// ------------------------------------------------------------------------------------------------ util
[[noreturn]] static void fatal(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vfprintf(stderr, fmt, ap);
    va_end(ap);
    fputc('\n', stderr);
    exit(code);
}

static void glck(gl_ctx* ctx, int rc, const char* what) {
    if (rc != GL_OK) fatal(1, "%s: %s", what, gl_last_error(ctx));
}

static double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
extern "C" int glhost_pool_size(void);              // libgoleft_b200.so: size of the host thread pool (creates it)
static void glhost_pool_warm() { (void)glhost_pool_size(); }

// Go's fmt spells non-finite floats "NaN", "+Inf", "-Inf" (C prints nan / inf): a sample with no tiles on a chromosome
// gets 0/0 in its ROC and bins.out / bins.in can be x/0, and parsers of .roc / .ped must see the reference's tokens.
static std::string go_float(const char* cfmt, double v) {
    if (std::isnan(v)) return "NaN";
    if (std::isinf(v)) return v > 0 ? "+Inf" : "-Inf";
    char b[64];
    snprintf(b, sizeof b, cfmt, v);
    return b;
}

static bool ends_with(const std::string& s, const std::string& suf) {
    return s.size() >= suf.size() && s.compare(s.size() - suf.size(), suf.size(), suf) == 0;
}

static bool file_exists(const std::string& p) { struct stat st; return stat(p.c_str(), &st) == 0; }

// lines of a (possibly gzipped) text file; like Go's ReadString('\n') loops that break on io.EOF, a final
// line WITHOUT a trailing newline is dropped when drop_unterminated is set (depth.go:106-110,137-141)
static std::vector<std::string> read_lines(const std::string& path, bool drop_unterminated) {
    gzFile f = gzopen(path.c_str(), "rb");
    if (!f) fatal(1, "open %s: %s", path.c_str(), strerror(errno));
    std::vector<std::string> out;
    std::string cur;
    char buf[1 << 16];
    int n;
    while ((n = gzread(f, buf, sizeof buf)) > 0) {
        for (int i = 0; i < n; i++) {
            if (buf[i] == '\n') { out.push_back(cur); cur.clear(); }
            else cur.push_back(buf[i]);
        }
    }
    gzclose(f);
    if (!cur.empty() && !drop_unterminated) out.push_back(cur);
    return out;
}

// go-arg style parser (alexflint/go-arg v1.4.3): -x v, --long v, --long=v, -long v; bool flags take no value
struct Spec { std::string lng; char sht; bool is_bool; std::string* sval; bool* bval; bool required; bool seen; };
struct ArgParser {
    std::string prog;
    std::vector<Spec> specs;
    std::vector<std::string> positional;
    void add(const std::string& lng, char sht, std::string* v, bool required = false) { specs.push_back({lng, sht, false, v, nullptr, required, false}); }
    void addb(const std::string& lng, char sht, bool* v) { specs.push_back({lng, sht, true, nullptr, v, false, false}); }
    bool given(const std::string& lng) const {
        for (const Spec& s : specs) if (s.lng == lng) return s.seen;
        return false;
    }
    [[noreturn]] void fail(const std::string& msg) const {
        fprintf(stderr, "Usage: %s [options] ...\nerror: %s\n", prog.c_str(), msg.c_str());
        exit(255);                                         // functional-tests.sh:40-42
    }
    void parse(int argc, char** argv) {
        for (int i = 1; i < argc; i++) {
            std::string a = argv[i];
            if (a == "-h" || a == "--help") {
                printf("Usage: %s", prog.c_str());
                for (auto& s : specs) printf(" [--%s%s]", s.lng.c_str(), s.is_bool ? "" : " VALUE");
                printf(" ...\n");
                exit(0);
            }
            if (a.size() > 1 && a[0] == '-' && !(a.size() > 1 && isdigit((unsigned char)a[1]))) {
                std::string name = a.substr(a[1] == '-' ? 2 : 1), val;
                bool has_val = false;
                size_t eq = name.find('=');
                if (eq != std::string::npos) { val = name.substr(eq + 1); name = name.substr(0, eq); has_val = true; }
                Spec* sp = nullptr;
                for (auto& s : specs) if (s.lng == name || (name.size() == 1 && s.sht && s.sht == name[0])) sp = &s;
                if (!sp) fail("unknown argument " + a);
                sp->seen = true;
                if (sp->is_bool) { *sp->bval = has_val ? (val == "true" || val == "1") : true; continue; }
                if (!has_val) {
                    if (i + 1 >= argc) fail("missing value for " + a);
                    val = argv[++i];
                }
                *sp->sval = val;
            } else {
                positional.push_back(a);
            }
        }
        for (auto& s : specs) if (s.required && !s.seen) fail(s.lng + " is required");
    }
};

// depth.go:73-94: regexp "(.+?)[:\t](\d+)([\-\t])(\d+).*?" — leftmost match, lazy first group
static bool chrom_start_end(const std::string& line, std::string& chrom, long long& start, long long& end) {
    const size_t n = line.size();
    for (size_t m0 = 0; m0 < n; m0++) {
        for (size_t k = m0 + 1; k < n; k++) {
            if (line[k] != ':' && line[k] != '\t') continue;
            size_t b = k + 1;
            while (b < n && isdigit((unsigned char)line[b])) b++;
            if (b == k + 1 || b >= n || (line[b] != '-' && line[b] != '\t')) continue;
            size_t d = b + 1;
            while (d < n && isdigit((unsigned char)line[d])) d++;
            if (d == b + 1) continue;
            chrom = line.substr(m0, k - m0);
            long long s = atoll(line.c_str() + k + 1);
            if (line[b] == '-') s--;
            start = s < 0 ? 0 : s;
            end = atoll(line.c_str() + b + 1);
            return true;
        }
    }
    return false;
}

// ------------------------------------------------------------------------------------------------ shared by the subcommands
static gl_ctx* open_ctx(int device, const char* prog) {
    gl_ctx* ctx = nullptr;
    if (gl_ctx_create(device, &ctx) != GL_OK) fatal(1, "%s: %s", prog, gl_last_error(nullptr));
    return ctx;
}

// --gpus: 0, or more than the visible devices, means one worker per device.  GL_OVERSUBSCRIBE (a testing aid) keeps the
// asked-for count on fewer devices: worker g runs on device g % n_dev.  There are never more workers than units of work.
struct GpuPlan { int G, n_dev; };
static GpuPlan resolve_gpus(const std::string& flag, size_t units, const char* prog) {
    int n_dev = 0;
    if (gl_device_count(&n_dev) != GL_OK || n_dev < 1) fatal(1, "%s: %s", prog, gl_last_error(nullptr));
    int G = atoi(flag.c_str());
    if (G <= 0 || (G > n_dev && !getenv("GL_OVERSUBSCRIBE"))) G = n_dev;
    G = (int)std::min<size_t>((size_t)G, std::max<size_t>(units, 1));
    return {G, n_dev};
}

// One host thread per worker, running fn(g).  With several GPUs each thread is bound to the NUMA node of its device; the
// host pool is created first, so that it keeps every core.
static std::vector<std::thread> start_workers(const GpuPlan& p, const std::function<void(int)>& fn) {
    glhost_pool_warm();
    std::vector<std::thread> th;
    for (int g = 0; g < p.G; g++)
        th.emplace_back([p, fn, g] {
            int node = -1, ncpu = 0;
            if (p.G > 1) gl_bind_numa_for_device(g % p.n_dev, 0, 1, &node, &ncpu);
            fn(g);
        });
    return th;
}

// A cohort's BAMs run by one worker per GPU and committed in argument order (covstats and depthwed from BAMs).  A worker
// claims the BAMs in argument order and opens the one after its current BAM before it runs the current one, so that the open
// overlaps the run.  No BAM after the first known failure is claimed, and one claimed ahead of a failure is closed without
// running.  The main thread takes the jobs in order with wait(i), and stop() joins the workers before a failure ends the run,
// so the failure reported is the first in argument order.
struct BamJob {
    gl_bam* bh = nullptr;
    bool done = false;
    int code = 0;                           // exit code of this BAM's failure (0: none) and its message
    std::string msg;
};

template <class Job> struct BamQueue {
    const std::vector<std::string>& bams;
    std::vector<Job> jobs;
    std::mutex mu;
    std::condition_variable cv;
    std::string setup_err;                  // the first worker that could not be set up: the message that ends the run
    size_t next_claim = 0, fail_at;         // no BAM after the first known failure is claimed
    std::vector<std::thread> th;

    explicit BamQueue(const std::vector<std::string>& b) : bams(b), jobs(b.size()), fail_at(b.size()) {}
    ~BamQueue() { stop(); }

    // Worker g: state = setup(g, err), where a message in err ends the run; run(state, i, next) for each BAM i it claims that
    // opened, next being the BAM opened after it (or null); teardown(state) at its end, set up or not.
    template <class Setup, class Run, class Teardown> void start(const GpuPlan& gp, Setup setup, Run run, Teardown teardown) {
        th = start_workers(gp, [this, setup, run, teardown](int g) {
            std::string err;
            auto st = setup(g, err);
            if (!err.empty()) {
                std::lock_guard<std::mutex> lk(mu);
                if (setup_err.empty()) setup_err = err;
                cv.notify_all();
            }
            const size_t S = jobs.size();
            for (size_t cur = err.empty() ? claim() : S; cur < S;) {
                if (behind(cur)) { close(cur); break; }
                const size_t nxt = claim();
                if (!jobs[cur].code) run(st, cur, nxt < S ? jobs[nxt].bh : nullptr);
                close(cur);
                std::lock_guard<std::mutex> lk(mu);
                jobs[cur].done = true;
                if (jobs[cur].code) fail_at = std::min(fail_at, cur);
                cv.notify_all();
                cur = nxt;
            }
            teardown(st);
        });
    }

    // the next BAM, opened (a failed open is its job's failure), or jobs.size() once claiming has ended
    size_t claim() {
        size_t i;
        {
            std::lock_guard<std::mutex> lk(mu);
            if (next_claim >= fail_at || !setup_err.empty()) return jobs.size();
            i = next_claim++;
        }
        char oerr[512] = {0};
        if (gl_bam_open(bams[i].c_str(), &jobs[i].bh, oerr, sizeof oerr) != GL_OK) { jobs[i].code = 1; jobs[i].msg = oerr; jobs[i].bh = nullptr; }
        return i;
    }

    // whether BAM i will never be committed: a BAM before it failed, or a worker could not be set up
    bool behind(size_t i) {
        std::lock_guard<std::mutex> lk(mu);
        return i > fail_at || !setup_err.empty();
    }

    void close(size_t i) {
        if (jobs[i].bh) gl_bam_close(jobs[i].bh);
        jobs[i].bh = nullptr;
    }

    // job i once its worker is done with it; a worker that could not be set up ends the run here instead
    Job& wait(size_t i) {
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [&] { return jobs[i].done || !setup_err.empty(); });
        if (!jobs[i].done) { lk.unlock(); stop(); fatal(1, "%s", setup_err.c_str()); }
        return jobs[i];
    }

    // ends the claiming and joins the workers
    void stop() {
        { std::lock_guard<std::mutex> lk(mu); fail_at = 0; }
        for (std::thread& t : th) t.join();
        th.clear();
    }
};

// whether a BAM's index can be seeked with: a stub index (stats bin but an empty / all-zero linear index for a reference that
// has reads) cannot, and such a BAM is decoded whole
static bool index_usable(const glhts::BamFile& f) {
    bool usable = f.has_index;
    for (size_t r = 0; usable && r < f.bai.ioffsets.size(); r++) {
        if (!f.bai.has_stats[r] || f.bai.mapped[r] + f.bai.unmapped[r] == 0) continue;
        bool any = false;
        for (uint64_t v : f.bai.ioffsets[r]) if (v) { any = true; break; }
        usable = any;
    }
    return usable;
}

// A BAM without a usable index cannot be seeked, so it is decoded once, whole, on `threads` host threads: reference `only`, or
// every reference for -1, into `whole`, which a SegSource then views.  True when it was, after `note` (when given) went to
// stderr; err then holds a failed decode's message.  False, with nothing decoded, for a BAM whose index can be used.
static bool decode_unindexed(const glhts::BamFile& f, const std::string& path, int Q, int threads, int only, glhts::SegmentSet& whole,
                             std::string& err, const char* note = nullptr) {
    if (index_usable(f)) return false;
    if (note) fprintf(stderr, "%s\n", note);
    err = glhts::bam_decode_segments(path, Q, threads, only, whole);
    return true;
}

// The bases of one pass over a contig: whole `step` chunks within the 2^30 - 1 bases the GPU reduces at once.  A window wider
// than that leaves no pass, and ends the run.
static long long pass_length(long long step, int W, const char* prog) {
    const long long n = ((1LL << 30) - 1) / step * step;
    if (n == 0) fatal(1, "%s: windowsize %d is above the 2^30 - 1 bases of one pass", prog, W);
    return n;
}

// the index of an input (indexcov.go:500-510): a .bai or .csi names itself; else the first of x.bam.bai, x.bai, x.bam.csi,
// x.csi that exists (BamFile::open's order), and when none does the x.bai whose read error the caller reports
static std::string bai_path(const std::string& b) {
    if (ends_with(b, ".csi")) return b;
    if (ends_with(b, ".bai")) return file_exists(b) ? b : b.substr(0, b.size() - 4);
    for (const std::string& p : glhts::index_candidates(b)) if (file_exists(p)) return p;
    return b.substr(0, b.size() - 4) + ".bai";
}

// indexcov and indexsplit size 16384-base tiles: a CSI whose tiles are wider cannot give them
static void refuse_wide_csi(const glhts::BaiIndex& idx, const std::string& path, const char* prog) {
    if (idx.is_csi && idx.min_shift > 14)
        fatal(1, "%s: %s is a CSI with min_shift %d: its tiles are wider than the 16384 bases indexcov sizes (min_shift 14 or less is needed)",
              prog, path.c_str(), idx.min_shift);
}

// CRAM pseudo-tile sizes of every reference of a .crai (crai.go:56-127), concatenated; ref_ptr[r] is where reference r's begin
static void crai_sizes(const std::vector<glhts::CraiSlices>& cr, std::vector<int64_t>& sizes, std::vector<int64_t>& ref_ptr) {
    sizes.clear();
    ref_ptr.assign(cr.size() + 1, 0);
    for (size_t r = 0; r < cr.size(); r++) {
        std::vector<int64_t> one;
        if (!glhts::crai_make_sizes(cr[r].start.data(), cr[r].span.data(), cr[r].bytes.data(), (int64_t)cr[r].start.size(), one))
            fatal(2, "panic: tilewidth logic error");
        sizes.insert(sizes.end(), one.begin(), one.end());
        ref_ptr[r + 1] = (int64_t)sizes.size();
    }
}

// One reference's segments, in the form they came in: packed8 words or int32 sorted by start from the host feeder (`host`),
// the GPU feeder's int32 arrays left on the device, or a host int32 view of a whole-file decode (or of any arrays the caller
// keeps alive).  Every int32 form is (s, e, n); packed8 words are read from `host`.
struct SegSource {
    glhts::ContigSegs host;
    const int32_t* s = nullptr; const int32_t* e = nullptr; int64_t n = 0;
    bool on_device = false;
    const glhts::SegmentSet* whole = nullptr;       // set for a BAM without a usable index: fetch views its decode, per tid

    // GL_GPU_FEED=0 keeps every decode on the host feeder
    static bool gpu_feed() {
        static const bool on = [] { const char* v = getenv("GL_GPU_FEED"); return !v || atoi(v) != 0; }();
        return on;
    }

    void view(const int32_t* vs, const int32_t* ve, int64_t vn) {
        host = glhts::ContigSegs();
        s = vs; e = ve; n = vn; on_device = false;
    }

    // the segments of reference tid (-1: not in the BAM, none) that can overlap [beg,end).  want: 0 auto, 32 int32.
    // whole_ref = the complete reference is wanted: the GPU feeder (BGZF inflate + record parse on the device, only compressed
    // bytes over PCIe) takes it when it can and GL_GPU_FEED allows; otherwise the host feeder decodes.  The decode's
    // statistics are added to *st, and a GPU-fed decode counts in *gpu_fed (both may be null).
    void fetch(gl_ctx* ctx, gl_bam& bam, int tid, long long beg, long long end, int Q, int threads, int want, bool whole_ref,
               glhts::DecodeStats* st, int* gpu_fed) {
        view(nullptr, nullptr, 0);
        if (tid < 0) return;
        if (whole) {
            const std::vector<int32_t>& ws = whole->start[(size_t)tid];
            view(ws.data(), whole->end[(size_t)tid].data(), (int64_t)ws.size());
            return;
        }
        glhts::DecodeStats one;
        if (whole_ref && gpu_feed()) {
            gl_bam_segments g;
            const int rc = gl_bam_decode_device(ctx, &bam, tid, Q, &s, &e, &n, &g);
            if (device_result(ctx, rc, g, "gl_bam_decode_device", one) && gpu_fed) ++*gpu_fed;
        }
        if (!on_device) {
            std::string err = bam.f.decode(tid, beg, end, Q, threads, want, host, &one);
            if (!err.empty()) fatal(1, "%s", err.c_str());
            if (host.format == 32) { s = host.start.data(); e = host.end.data(); n = host.n; }
        }
        add_stats(st, one);
    }

    // The segments of reference tid whose blocks meet one of the intervals [beg[i], end[i]), decoded on the device from only
    // the BGZF members the index's bin query names; they stay on the device.  False, with nothing fetched, where the GPU
    // feeder cannot serve them (GL_GPU_FEED=0, a preloaded BAM, or GL_ESTATE from the library): the caller uses fetch().
    bool fetch_regions(gl_ctx* ctx, gl_bam& bam, int tid, const std::vector<int64_t>& beg, const std::vector<int64_t>& end, int Q,
                       glhts::DecodeStats* st) {
        view(nullptr, nullptr, 0);
        if (tid < 0 || whole || !gpu_feed()) return false;
        glhts::DecodeStats one;
        gl_bam_segments g;
        const int rc = gl_bam_decode_device_regions(ctx, &bam, tid, beg.data(), end.data(), (int64_t)beg.size(), Q, &s, &e, &n, &g);
        if (!device_result(ctx, rc, g, "gl_bam_decode_device_regions", one)) return false;
        add_stats(st, one);
        return true;
    }

    // One pass [ps, pe) over reference tid, of length len: a region query on the GPU feeder when the pass is not the whole
    // reference and the feeder serves it (only a CSI can index past 2^29), else fetch().  A GPU-fed pass counts in *gpu_fed.
    void fetch_pass(gl_ctx* ctx, gl_bam& bam, int tid, long long ps, long long pe, long long len, int Q, int threads,
                    glhts::DecodeStats* st, int* gpu_fed) {
        const bool whole_ref = ps == 0 && pe == len;
        if (!whole_ref && fetch_regions(ctx, bam, tid, {ps}, {pe}, Q, st)) ++*gpu_fed;
        else fetch(ctx, bam, tid, ps, pe, Q, threads, 0, whole_ref, st, gpu_fed);
    }

    // a device decode's outcome: on GL_OK the arrays are on the device and its statistics go to one; GL_ESTATE (not possible
    // on the device for this reference) leaves nothing; any other code is fatal
    bool device_result(gl_ctx* ctx, int rc, const gl_bam_segments& g, const char* what, glhts::DecodeStats& one) {
        if (rc != GL_OK) {
            view(nullptr, nullptr, 0);
            if (rc != GL_ESTATE) glck(ctx, rc, what);
            return false;
        }
        on_device = true;
        one.wall_s = g.wall_s; one.inflate_s = g.inflate_s; one.parse_s = g.parse_s;
        one.n_records = g.n_records; one.bytes_in = g.bytes_in; one.bytes_out = g.bytes_out;
        return true;
    }

    static void add_stats(glhts::DecodeStats* st, const glhts::DecodeStats& one) {
        if (!st) return;
        st->wall_s += one.wall_s; st->inflate_s += one.inflate_s; st->parse_s += one.parse_s;
        st->n_records += one.n_records; st->bytes_in += one.bytes_in; st->bytes_out += one.bytes_out;
    }

    void add(gl_ctx* ctx) const {
        if (host.format == 8) {
            if (host.n_blocks > 0)
                glck(ctx, gl_depth_add_segments_packed8(ctx, host.anchors.data(), host.ds.data(), host.len.data(), host.n_blocks), "gl_depth_add_segments_packed8");
        } else if (n > 0) {
            if (on_device) glck(ctx, gl_depth_add_segments_device(ctx, s, e, n), "gl_depth_add_segments_device");
            else glck(ctx, gl_depth_add_segments(ctx, s, e, n), "gl_depth_add_segments");
        }
    }
};

// A FASTA opened for Faidx.Stats (github.com/brentp/faidx, restated in fasta.cu): its .fai records and its bytes, mapped.
// `depth --stats` and `dcnv` take the GC of their rows through it.
struct FastaStats {
    std::vector<glhts::RefInfo> index;
    const uint8_t* map = nullptr; size_t len = 0;
    FastaStats() = default;
    FastaStats(const FastaStats&) = delete;
    FastaStats& operator=(const FastaStats&) = delete;
    ~FastaStats() { if (map) munmap(const_cast<uint8_t*>(map), len); }
    void open(const std::string& path) {
        std::string e = glhts::fai_read(path + ".fai", index);
        if (!e.empty()) fatal(1, "%s", e.c_str());
        int fd = ::open(path.c_str(), O_RDONLY);
        struct stat st;
        if (fd < 0 || fstat(fd, &st) != 0) fatal(1, "cannot open %s", path.c_str());
        len = (size_t)st.st_size;
        if (len) {
            void* mm = mmap(nullptr, len, PROT_READ, MAP_PRIVATE, fd, 0);
            if (mm == MAP_FAILED) fatal(1, "cannot mmap %s", path.c_str());
            map = static_cast<const uint8_t*>(mm);
        }
        close(fd);
    }
    const glhts::RefInfo* find(const std::string& c) const {
        for (const glhts::RefInfo& r : index) if (r.name == c) return &r;
        return nullptr;
    }
    // {GC, CpG, Masked} of the rows [s[i], e[i]) of one record into st3[3 i ..] (one gl_fasta_load, one gl_fasta_stats).
    // Faidx.Stats panics on a row outside the record (s < 0, e < s or e > length); such a row is clipped to the record
    // here and counted in the return value, and each caller decides what that means.
    size_t stats(gl_ctx* ctx, const glhts::RefInfo& ri, const std::vector<int64_t>& s, const std::vector<int64_t>& e, double* st3) const {
        if (s.empty()) return 0;
        const int64_t rec_bytes = std::min<int64_t>((int64_t)len - ri.offset, glhts::fasta_position(ri, ri.length) + 1);
        if (ri.offset < 0 || rec_bytes < 0) fatal(1, "bad .fai entry for %s", ri.name.c_str());
        glck(ctx, gl_fasta_load(ctx, map + ri.offset, rec_bytes), "gl_fasta_load");
        std::vector<int64_t> ba(s.size()), bb(s.size());
        size_t outside = 0;
        for (size_t i = 0; i < s.size(); i++) {
            outside += (s[i] < 0 || e[i] < s[i] || e[i] > ri.length);
            const int64_t a = std::min<int64_t>(std::max<int64_t>(s[i], 0), ri.length), b = std::min<int64_t>(std::max<int64_t>(e[i], a), ri.length);
            const int64_t ps = glhts::fasta_position(ri, a), pe = glhts::fasta_position(ri, b);
            ba[i] = std::min(ps, rec_bytes);          // the slice ends one byte past position(end) when that byte exists
            bb[i] = std::max(ba[i], std::min<int64_t>(pe + ((ri.offset + pe < (int64_t)len) ? 1 : 0), rec_bytes));
        }
        glck(ctx, gl_fasta_stats(ctx, ba.data(), bb.data(), (int64_t)ba.size(), nullptr, st3), "gl_fasta_stats");
        return outside;
    }
};

// ------------------------------------------------------------------------------------------------ depth
// `goleft depth`: depth/depth.go:103-159 builds the work list (10 Mb chunks of every .fai contig, or the BED lines), runs one
// `samtools depth -r` child per entry and concatenates the per-chunk BED files (-o: in order).  Here the unit of work is a
// contig (all its chunks in one GPU pass, run_break = step keeps the per-chunk row structure) or, in BED mode, a contig's
// BED lines; contigs are dealt to the visible GPUs longest first (gl_lpt_assign), one host thread + one gl_ctx + one BAM
// handle per GPU; the host pool (inflate + parse) is shared.  Output is always in work-list order (a valid -o output).
namespace {

struct DepthOpts {
    int W = 250, maxmean = 0, Q = 1, mincov = 4, threads = 0;
    long long step = 10000000;
    long long pass = 0;                             // .fai mode: the bases of one GPU pass (pass_length)
    bool stats = false;
    std::string reference;
};

struct DepthRegion { std::string chrom; long long s, e; };

struct DepthJob {                                   // one contig (.fai mode) or the BED lines of one contig (BED mode)
    std::string chrom;
    long long len = 0;                              // .fai mode: contig length
    std::vector<size_t> lines;                      // BED mode: indices into the region list
    std::string hd, ca;                             // .fai mode output
    glhts::DecodeStats dec;                         // summed over the job's decodes
    double gpu_s = 0;
    int gpu_fed = 0;                                // passes whose segments came from the GPU feeder
    bool done = false;
};

struct DepthShared {
    const DepthOpts* opt;
    std::string bam_path;
    const glhts::SegmentSet* preload = nullptr;     // BAM without an index: every contig decoded once up front
    std::vector<DepthRegion>* regions = nullptr;    // BED mode
    std::vector<std::string>* out_hd = nullptr;     // BED mode: per line
    std::vector<std::string>* out_ca = nullptr;
    FastaStats fa;                                  // --stats
    std::mutex mu; std::condition_variable cv;
};

// One GPU's worker: ctx + BAM handle + buffers
struct DepthEngine {
    DepthShared& sh;
    const DepthOpts& o;
    gl_ctx* ctx = nullptr;
    gl_bam gbam;                                            // the library's BAM handle (host and GPU feeder)
    std::map<std::string, int> tid_of;
    SegSource src;
    std::vector<int64_t> sums; std::vector<int32_t> rstart; std::vector<uint8_t> rclass;
    std::vector<char> tbuf_hd, tbuf_ca;
    // --stats state (depth.go:191-200,246-252): chunks of a contig are parked, one gl_fasta_stats launch for all their rows
    struct Pending { std::string chrom; long long rs, re; std::vector<int64_t> sums; std::vector<int32_t> rs_; std::vector<uint8_t> rc_; std::string *hd, *ca; int64_t row0, nrows; };
    std::vector<Pending> pending;
    std::vector<int64_t> row_s, row_e;

    DepthEngine(DepthShared& s, int device) : sh(s), o(*s.opt) {
        ctx = open_ctx(device, "goleft depth");
        if (sh.preload) {
            src.whole = sh.preload;
        } else {
            std::string e = gbam.f.open(sh.bam_path);
            if (!e.empty()) fatal(1, "%s", e.c_str());
        }
        const glhts::BamHeader& hdr = sh.preload ? sh.preload->header : gbam.f.header;
        for (size_t i = 0; i < hdr.refs.size(); i++) tid_of[hdr.refs[i].name] = (int)i;
        rstart.resize(1 << 16); rclass.resize(1 << 16);
    }
    ~DepthEngine() { gl_ctx_destroy(ctx); }

    int tid(const std::string& c) const { auto it = tid_of.find(c); return it == tid_of.end() ? -1 : it->second; }

    // window sums + class runs of [rs,re) on the host (the --stats and BED paths)
    void reduce_to_host(const SegSource& segs, long long rs, long long re, long long run_break, int64_t& nw, int64_t& nr) {
        glck(ctx, gl_depth_begin(ctx, rs, re), "gl_depth_begin");
        segs.add(ctx);
        glck(ctx, gl_depth_reduce(ctx, o.W, o.mincov, o.maxmean, run_break), "gl_depth_reduce");
        int32_t md = 0;
        glck(ctx, gl_depth_result_sizes(ctx, &nw, &nr, &md), "gl_depth_result_sizes");
        sums.resize((size_t)nw);
        if ((int64_t)rstart.size() < nr) { rstart.resize((size_t)nr + 1024); rclass.resize((size_t)nr + 1024); }
        glck(ctx, gl_depth_get_windows(ctx, sums.data(), nw), "gl_depth_get_windows");
        glck(ctx, gl_depth_get_runs(ctx, rstart.data(), nullptr, rclass.data(), (int64_t)rstart.size()), "gl_depth_get_runs");
    }

    void emit(const std::string& c, long long rs, long long re, const int64_t* ws, int64_t nw, const int32_t* rs_, const uint8_t* rc_, int64_t nr,
              std::string* hd_to, std::string* ca_to) {
        if (!o.stats) {
            char *hd = nullptr, *ca = nullptr;
            int64_t hl = 0, cl = 0;
            if (gl_depth_format_chunk(c.c_str(), rs, re, o.W, ws, nw, rs_, rc_, nr, &hd, &hl, &ca, &cl) != GL_OK) fatal(1, "gl_depth_format_chunk failed");
            hd_to->append(hd, (size_t)hl); ca_to->append(ca, (size_t)cl);
            gl_free_text(hd); gl_free_text(ca);
            return;
        }
        Pending pc{c, rs, re, std::vector<int64_t>(ws, ws + nw), std::vector<int32_t>(rs_, rs_ + nr), std::vector<uint8_t>(rc_, rc_ + nr), hd_to, ca_to,
                   (int64_t)row_s.size(), 0};
        int64_t n = 0;
        gl_depth_chunk_rows(rs, re, o.W, rs_, rc_, nr, nullptr, nullptr, 0, &n);
        row_s.resize(row_s.size() + (size_t)n); row_e.resize(row_s.size());
        if (gl_depth_chunk_rows(rs, re, o.W, rs_, rc_, nr, row_s.data() + pc.row0, row_e.data() + pc.row0, n, &n) != GL_OK) fatal(1, "gl_depth_chunk_rows failed");
        pc.nrows = n;
        pending.push_back(std::move(pc));
    }

    void flush_stats() {                                    // all parked chunks belong to one contig
        if (pending.empty()) return;
        const std::string& c = pending[0].chrom;
        std::vector<double> st3(row_s.size() * 3, 0.0);
        const glhts::RefInfo* ri = sh.fa.find(c);
        if (!ri) fprintf(stderr, "GC: unknown sequence %s\n", c.c_str());                 // faidx error text; zeros are printed (depth.go:195-199)
        else sh.fa.stats(ctx, *ri, row_s, row_e, st3.data());                            // faidx panics past the contig; clipped here instead
        for (const Pending& pc : pending) {
            char *hd = nullptr, *ca = nullptr;
            int64_t hl = 0, cl = 0;
            if (gl_depth_format_chunk_stats(pc.chrom.c_str(), pc.rs, pc.re, o.W, pc.sums.data(), (int64_t)pc.sums.size(), pc.rs_.data(), pc.rc_.data(),
                                            (int64_t)pc.rs_.size(), st3.data() + pc.row0 * 3, pc.nrows, &hd, &hl, &ca, &cl) != GL_OK)
                fatal(1, "gl_depth_format_chunk_stats failed");
            pc.hd->append(hd, (size_t)hl); pc.ca->append(ca, (size_t)cl);
            gl_free_text(hd); gl_free_text(ca);
        }
        pending.clear(); row_s.clear(); row_e.clear();
    }

    // BED text of [ps,pe) made on the device by call(depth_bed, cap, &len, callable_bed, cap, &len), appended to the job.  The
    // buffers start at gl_depth_text_bound's size; a call that reports GL_ERANGE has set the lengths it needs and runs once more.
    template <class Call> void device_text(DepthJob& job, long long ps, long long pe, const char* what, Call call) {
        const int64_t nwin = (pe - 1) / o.W - ps / o.W + 1;
        const size_t need_hd = (size_t)gl_depth_text_bound(job.chrom.c_str(), nwin);
        if (tbuf_hd.size() < need_hd) tbuf_hd.resize(need_hd);
        if (tbuf_ca.size() < (size_t)(1 << 20)) tbuf_ca.resize(1 << 20);
        int64_t hl = 0, cl = 0;
        int rc = call(tbuf_hd.data(), (int64_t)tbuf_hd.size(), &hl, tbuf_ca.data(), (int64_t)tbuf_ca.size(), &cl);
        if (rc == GL_ERANGE) {
            tbuf_hd.resize((size_t)hl + 16); tbuf_ca.resize((size_t)cl + 16);
            rc = call(tbuf_hd.data(), (int64_t)tbuf_hd.size(), &hl, tbuf_ca.data(), (int64_t)tbuf_ca.size(), &cl);
        }
        glck(ctx, rc, what);
        job.hd.append(tbuf_hd.data(), (size_t)hl);
        job.ca.append(tbuf_ca.data(), (size_t)cl);
    }

    // ---- .fai mode: one contig, in passes of o.pass bases whose texts concatenate (chunk edges are run breaks anyway)
    void run_contig(DepthJob& job) {
        const char* c = job.chrom.c_str();
        for (long long ps = 0; ps < job.len; ps += o.pass) {
            const long long pe = std::min(job.len, ps + o.pass);
            src.fetch_pass(ctx, gbam, tid(job.chrom), ps, pe, job.len, o.Q, o.threads, &job.dec, &job.gpu_fed);
            const double tg = now_s();
            const bool dtext = !o.stats && job.chrom.size() <= 64;
            if (dtext && src.on_device) {                                      // segments already on the device (GPU feeder)
                glck(ctx, gl_depth_begin(ctx, ps, pe), "gl_depth_begin");
                src.add(ctx);
                glck(ctx, gl_depth_reduce(ctx, o.W, o.mincov, o.maxmean, o.step), "gl_depth_reduce");
                device_text(job, ps, pe, "gl_depth_text", [&](char* hd, int64_t hc, int64_t* hl, char* ca, int64_t cc, int64_t* cl) {
                    return gl_depth_text(ctx, c, hd, hc, hl, ca, cc, cl);
                });
            } else if (dtext) {                                                // host segments: the library picks the transport
                device_text(job, ps, pe, "gl_depth_bed_region", [&](char* hd, int64_t hc, int64_t* hl, char* ca, int64_t cc, int64_t* cl) {
                    const glhts::ContigSegs& h = src.host;
                    if (h.format == 8)
                        return gl_depth_bed_region_packed8(ctx, c, ps, pe, h.anchors.data(), h.ds.data(), h.len.data(), h.n_blocks, o.W, o.mincov,
                                                           o.maxmean, o.step, hd, hc, hl, ca, cc, cl);
                    return gl_depth_bed_region(ctx, c, ps, pe, src.s, src.e, src.n, o.W, o.mincov, o.maxmean, o.step, o.threads, hd, hc, hl, ca, cc, cl);
                });
            } else {
                int64_t nw = 0, nr = 0;
                reduce_to_host(src, ps, pe, o.step, nw, nr);
                for (long long cs = ps; cs < pe; cs += o.step) {
                    const long long ce = std::min(cs + o.step, pe);
                    const int32_t* lo = std::lower_bound(rstart.data(), rstart.data() + nr, (int32_t)cs);
                    const int32_t* hi = std::lower_bound(rstart.data(), rstart.data() + nr, (int32_t)ce);
                    emit(job.chrom, cs, ce, sums.data() + (cs / o.W - ps / o.W), (ce - 1) / o.W - cs / o.W + 1, lo, rclass.data() + (lo - rstart.data()), hi - lo,
                         &job.hd, &job.ca);
                }
                flush_stats();
            }
            job.gpu_s += now_s() - tg;
        }
    }

    // ---- BED mode: the lines of one contig.  One pass over the span they cover (window sums + class runs, run_break 0),
    //      the clipped first/last window of every line from gl_depth_interval_sums, then the reference's rows line by line
    //      (depth.go:293-358 sees each line as its own chunk).
    void run_bed_chrom(DepthJob& job) {
        std::vector<DepthRegion>& regions = *sh.regions;
        const std::vector<size_t>& ks = job.lines;
        const int W = o.W;
        long long lo = regions[ks[0]].s, hi = regions[ks[0]].e;
        for (size_t k : ks) { lo = std::min(lo, regions[k].s); hi = std::max(hi, regions[k].e); }
        const long long span_s = lo / W * W;
        const int t = tid(job.chrom);
        int64_t nw = 0, nr = 0;
        auto format_one = [&](size_t k, const int64_t* ws, int64_t nw_, const int32_t* rs_, const uint8_t* rc_, int64_t nr_) {
            emit(regions[k].chrom, regions[k].s, regions[k].e, ws, nw_, rs_, rc_, nr_, &(*sh.out_hd)[k], &(*sh.out_ca)[k]);
        };
        bool batched = ks.size() > 1 && hi - span_s < (1LL << 30) - 2 * (long long)W;
        // The GPU feeder reads only the members the lines' bin queries name.  Its blocks are those that meet a line, in BAM
        // order: what one pass over the span needs, or a single line's pass, but not the per-line slices of sorted arrays.
        bool dev = false;
        if (batched || ks.size() == 1) {
            std::vector<int64_t> lb, le;
            for (size_t k : ks) { lb.push_back(regions[k].s); le.push_back(regions[k].e); }
            dev = src.fetch_regions(ctx, gbam, t, lb, le, o.Q, &job.dec);
        }
        if (!dev) src.fetch(ctx, gbam, t, span_s, hi, o.Q, o.threads, 32, false, &job.dec, &job.gpu_fed);   // int32: the interval sums and the per-line slices want arrays
        const double tg = now_s();
        if (batched) {
            reduce_to_host(src, span_s, hi, 0, nw, nr);
            int32_t path = 0;
            batched = gl_depth_last_path(ctx, &path) == GL_OK && (path == 1 || src.n == 0);   // the interval sums want the fused path's cell index
            if (!batched && dev) {                                             // per-line passes slice sorted host arrays
                dev = false;
                src.fetch(ctx, gbam, t, span_s, hi, o.Q, o.threads, 32, false, &job.dec, &job.gpu_fed);
            }
        }
        if (dev) job.gpu_fed++;
        if (!batched) {
            // per-line passes over the slice of segments that can reach the line (the arrays are sorted by start)
            const int32_t maxlen = std::max<int32_t>(src.host.max_len, 1);
            const bool sorted = !sh.preload;                                   // the index-guided decoder sorts; preloaded arrays are in record order
            SegSource line;
            for (size_t k : ks) {
                if (regions[k].e - regions[k].s >= (1LL << 30)) fatal(1, "BED region longer than 2^30-1 bases: %s", regions[k].chrom.c_str());
                if (src.on_device) {                                           // one line, its blocks from the GPU feeder
                    reduce_to_host(src, regions[k].s, regions[k].e, 0, nw, nr);
                    format_one(k, sums.data(), nw, rstart.data(), rclass.data(), nr);
                    continue;
                }
                int64_t a = 0, b = src.n;
                if (sorted && src.n > 0) {
                    a = std::lower_bound(src.s, src.s + src.n, (int32_t)std::max<long long>(regions[k].s - maxlen, INT32_MIN)) - src.s;
                    b = std::lower_bound(src.s, src.s + src.n, (int32_t)std::min<long long>(regions[k].e, INT32_MAX)) - src.s;
                }
                line.view(src.s + a, src.e + a, b - a);
                reduce_to_host(line, regions[k].s, regions[k].e, 0, nw, nr);
                format_one(k, sums.data(), nw, rstart.data(), rclass.data(), nr);
            }
            flush_stats();
            job.gpu_s += now_s() - tg;
            return;
        }
        std::vector<int64_t> rsum, edge;
        std::vector<int32_t> ia, ib, rrs;
        std::vector<uint8_t> rrc;
        for (size_t k : ks) {                                            // clipped edge windows
            const long long s = regions[k].s, e = regions[k].e, w0 = s / W, w1 = (e - 1) / W;
            if (s % W != 0 || (w0 == w1 && e != (w0 + 1) * W)) { ia.push_back((int32_t)s); ib.push_back((int32_t)std::min(e, (w0 + 1) * W)); }
            if (w1 > w0 && e != (w1 + 1) * W) { ia.push_back((int32_t)(w1 * W)); ib.push_back((int32_t)e); }
        }
        edge.resize(ia.size());
        if (!ia.empty()) glck(ctx, gl_depth_interval_sums(ctx, ia.data(), ib.data(), (int64_t)ia.size(), edge.data()), "gl_depth_interval_sums");
        size_t ei = 0;
        const long long sw0 = span_s / W;
        for (size_t k : ks) {
            const long long s = regions[k].s, e = regions[k].e, w0 = s / W, w1 = (e - 1) / W;
            rsum.assign(sums.begin() + (w0 - sw0), sums.begin() + (w1 - sw0) + 1);
            if (s % W != 0 || (w0 == w1 && e != (w0 + 1) * W)) rsum[0] = edge[ei++];
            if (w1 > w0 && e != (w1 + 1) * W) rsum.back() = edge[ei++];
            const int32_t* rb = rstart.data();
            const int32_t* first = std::upper_bound(rb, rb + nr, (int32_t)s);          // first run starting after s
            const int32_t* last = std::lower_bound(rb, rb + nr, (int32_t)e);
            rrs.assign(1, (int32_t)s);
            rrc.assign(1, rclass[(size_t)(first - rb) - 1]);                           // run_start[0] == span_s <= s
            rrs.insert(rrs.end(), first, last);
            rrc.insert(rrc.end(), rclass.data() + (first - rb), rclass.data() + (last - rb));
            format_one(k, rsum.data(), (int64_t)rsum.size(), rrs.data(), rrc.data(), (int64_t)rrs.size());
        }
        flush_stats();
        job.gpu_s += now_s() - tg;
    }
};

}  // namespace

static int cmd_depth(int argc, char** argv) {
    std::string w = "250", m = "0", q = "1", chrom, mincov = "4", reference, procs = "0", bed, prefix, gpus = "0";
    bool ordered = false, stats = false, timing = false;
    ArgParser ap;
    ap.prog = "goleft depth";
    ap.add("windowsize", 'w', &w); ap.add("maxmeandepth", 'm', &m); ap.addb("ordered", 'o', &ordered);
    ap.add("q", 'Q', &q); ap.add("chrom", 'c', &chrom); ap.add("mincov", 0, &mincov); ap.addb("stats", 's', &stats);
    ap.add("reference", 'r', &reference); ap.add("processes", 'p', &procs); ap.add("bed", 'b', &bed);
    ap.add("prefix", 0, &prefix, true);
    ap.add("gpus", 0, &gpus);                       // extension: GPUs to use (0 = every visible one)
    ap.addb("timing", 0, &timing);                  // extension: per-phase wall clock on stderr
    ap.parse(argc, argv);
    if (ap.positional.empty()) ap.fail("bam is required");
    const std::string bam = ap.positional[0];
    DepthOpts o;
    o.W = atoi(w.c_str()); o.maxmean = atoi(m.c_str()); o.Q = atoi(q.c_str()); o.mincov = atoi(mincov.c_str());
    o.stats = stats; o.reference = reference;
    if (o.W <= 0) ap.fail("windowsize must be > 0");
    o.threads = atoi(procs.c_str());
    if (o.threads < 0) o.threads = 0;               // 0 = every thread of the host pool
    o.step = std::max(1LL, 10000000LL / o.W) * o.W;                          // depth.go:132
    const double t_start = now_s();

    // work list (depth.go:103-159)
    std::vector<DepthRegion> regions;
    std::vector<DepthJob> jobs;
    if (!bed.empty()) {
        for (const std::string& ln : read_lines(bed, true)) {
            if (ln.empty()) continue;
            DepthRegion r;
            if (!chrom_start_end(ln, r.chrom, r.s, r.e)) fatal(1, "couldn't get region from line%s", ln.c_str());
            regions.push_back(r);
        }
        std::map<std::string, size_t> job_of;
        for (size_t k = 0; k < regions.size(); k++) {
            if (regions[k].e <= regions[k].s) continue;
            auto ins = job_of.emplace(regions[k].chrom, jobs.size());
            if (ins.second) { jobs.emplace_back(); jobs.back().chrom = regions[k].chrom; }
            DepthJob& j = jobs[ins.first->second];
            j.lines.push_back(k);
            j.len = std::max(j.len, regions[k].e);
        }
    } else {
        for (const std::string& ln : read_lines(reference + ".fai", true)) {
            size_t t1 = ln.find('\t');
            if (t1 == std::string::npos) continue;
            std::string c = ln.substr(0, t1);
            if (!chrom.empty() && c != chrom) continue;
            const long long len = atoll(ln.c_str() + t1 + 1);
            if (len <= 0) continue;
            jobs.emplace_back();
            jobs.back().chrom = c; jobs.back().len = len;
        }
        if (!jobs.empty()) o.pass = pass_length(o.step, o.W, "goleft depth");
    }

    DepthShared sh;
    sh.opt = &o;
    sh.bam_path = bam;
    std::vector<std::string> out_hd(regions.size()), out_ca(regions.size());
    sh.regions = &regions; sh.out_hd = &out_hd; sh.out_ca = &out_ca;
    // an unindexed BAM is decoded once, whole (the reference's `samtools depth -r` would refuse it)
    glhts::SegmentSet preload;
    {
        glhts::BamFile probe;
        std::string e = probe.open(bam);
        if (!e.empty()) fatal(1, "%s", e.c_str());
        const int thr = o.threads > 0 ? o.threads : (int)std::max(1u, std::thread::hardware_concurrency());
        int only = -1;
        if (!chrom.empty()) for (size_t i = 0; i < probe.header.refs.size(); i++) if (probe.header.refs[i].name == chrom) only = (int)i;
        const std::string note = "goleft depth: no usable index (.bai or .csi) next to " + bam +
                                 ": decoding the whole file (index it for -c / --bed to read only what they need)";
        if (decode_unindexed(probe, bam, o.Q, thr, only, preload, e, note.c_str())) {
            if (!e.empty()) fatal(1, "%s", e.c_str());
            sh.preload = &preload;
        }
    }
    if (stats) {
        if (reference.empty()) fatal(1, "goleft depth: --stats needs --reference");
        sh.fa.open(reference);
    }

    const std::string sfx = chrom.empty() ? "" : "." + chrom;               // depth.go:378-389
    FILE* fca = fopen((prefix + sfx + ".callable.bed").c_str(), "w");
    FILE* fhd = fopen((prefix + sfx + ".depth.bed").c_str(), "w");
    if (!fca || !fhd) fatal(1, "cannot create output files with prefix %s", prefix.c_str());

    // ---- GPUs and placement
    const GpuPlan gp = resolve_gpus(gpus, jobs.size(), "goleft depth");
    std::vector<int32_t> gpu_of(jobs.size(), 0);
    {
        std::vector<int64_t> wts(jobs.size());
        for (size_t i = 0; i < jobs.size(); i++) wts[i] = jobs[i].len;
        if (!jobs.empty() && gl_lpt_assign(wts.data(), (int32_t)jobs.size(), gp.G, gpu_of.data(), nullptr) != GL_OK) fatal(1, "gl_lpt_assign failed");
    }
    std::vector<std::thread> th = start_workers(gp, [&](int g) {
        DepthEngine eng(sh, g % gp.n_dev);
        for (size_t i = 0; i < jobs.size(); i++) {
            if (gpu_of[i] != g) continue;
            if (bed.empty()) eng.run_contig(jobs[i]); else eng.run_bed_chrom(jobs[i]);
            { std::lock_guard<std::mutex> lk(sh.mu); jobs[i].done = true; }
            sh.cv.notify_all();
        }
    });
    // ---- ordered output as the jobs finish
    if (bed.empty()) {
        for (size_t i = 0; i < jobs.size(); i++) {
            { std::unique_lock<std::mutex> lk(sh.mu); sh.cv.wait(lk, [&] { return jobs[i].done; }); }
            fwrite(jobs[i].hd.data(), 1, jobs[i].hd.size(), fhd);
            fwrite(jobs[i].ca.data(), 1, jobs[i].ca.size(), fca);
            std::string().swap(jobs[i].hd); std::string().swap(jobs[i].ca);
        }
    }
    for (auto& t : th) t.join();
    if (!bed.empty()) {
        for (size_t k = 0; k < regions.size(); k++) {
            fwrite(out_hd[k].data(), 1, out_hd[k].size(), fhd);
            fwrite(out_ca[k].data(), 1, out_ca[k].size(), fca);
        }
    }
    fclose(fca); fclose(fhd);
    if (timing) {
        double dec = 0, gpu = 0, inf = 0, par = 0; long long rec = 0, bin = 0, bout = 0; int fed = 0;
        for (const DepthJob& j : jobs) {
            fed += j.gpu_fed; gpu += j.gpu_s;
            dec += j.dec.wall_s; inf += j.dec.inflate_s; par += j.dec.parse_s; rec += j.dec.n_records; bin += j.dec.bytes_in; bout += j.dec.bytes_out;
        }
        fprintf(stderr, "{\"goleft_depth_timing\": {\"wall_s\": %.4f, \"gpus\": %d, \"jobs\": %zu, \"decode_wall_s_sum\": %.4f, \"gpu_call_s_sum\": %.4f, "
                        "\"inflate_thread_s_sum\": %.4f, \"parse_thread_s_sum\": %.4f, "
                        "\"records\": %lld, \"bgzf_bytes_in\": %lld, \"bgzf_bytes_out\": %lld, \"host_threads\": %d, \"gpu_fed_passes\": %d}}\n",
                now_s() - t_start, gp.G, jobs.size(), dec, gpu, inf, par, rec, bin, bout, glhost_pool_size(), fed);
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------ indexcov
// indexcov.go:213-246
static std::string short_name(const std::string& b, bool from_filename, const glhts::BamHeader* hdr) {
    if (!from_filename && hdr) {
        std::vector<std::string> sm = hdr->sample_names();
        if (sm.size() > 1) fatal(1, "bam reagroup: more than one RG for %s", b.c_str());
        if (sm.size() == 1) return sm[0];
    }
    std::string v = b.substr(b.find_last_of('/') == std::string::npos ? 0 : b.find_last_of('/') + 1);
    std::vector<std::string> parts;
    size_t p = 0;
    for (;;) { size_t d = v.find('.', p); parts.push_back(v.substr(p, d == std::string::npos ? std::string::npos : d - p)); if (d == std::string::npos) break; p = d + 1; }
    if (parts.size() <= 2) return parts[0];
    std::string out = parts[0];
    for (size_t i = 1; i + 1 < parts.size(); i++) out += "-" + parts[i];
    return out;
}

// indexcov.go:530-547
static bool same_chrom(const std::vector<std::string>& as, const std::string& b) {
    for (const std::string& a : as) {
        if (a == b) return true;
        std::string na = a;
        if (a.compare(0, 3, "chr") == 0) na = a.substr(3);
        else if (b.compare(0, 3, "chr") == 0) na = "chr" + a;
        if (na == b) return true;
    }
    return false;
}

// indexcov.go:957-991 for one sample
static double get_cn(const float* d, size_t n) {
    std::vector<float> tmp;
    size_t lows = 0;
    for (size_t i = 0; i < n; i++) if (d[i] != 0) { tmp.push_back(d[i]); if (d[i] < 0.02f) lows++; }
    if (tmp.empty()) return -0.1;
    std::sort(tmp.begin(), tmp.end());
    const double pLo = (double)lows / (double)n;
    const float* t = tmp.data();
    size_t tk = tmp.size();
    if (pLo > 0.3) { t += lows; tk -= lows; }
    if (tk == 0) return 0;
    return (double)(2.0f * t[(size_t)((double)tk * 0.4)]);
}

struct IcRef { std::string name; long long len; int id; };

template <class T> struct RawBuf {                          // malloc'ed, uninitialised, sized once
    T* p = nullptr; size_t n = 0;
    RawBuf() = default;
    RawBuf(const RawBuf&) = delete;
    RawBuf& operator=(const RawBuf&) = delete;
    ~RawBuf() { free(p); }
    void resize(size_t m) { free(p); p = static_cast<T*>(malloc(std::max<size_t>(m, 1) * sizeof(T))); n = m; if (!p) fatal(1, "out of memory (%zu bytes)", m * sizeof(T)); }
    T* data() { return p; }
    T& operator[](size_t i) { return p[i]; }
};

// device buffers of one ctx, freed together when the owner goes out of scope
struct DevBufs {
    gl_ctx* ctx;
    std::vector<void*> ptrs;
    explicit DevBufs(gl_ctx* c = nullptr) : ctx(c) {}
    DevBufs(const DevBufs&) = delete;
    DevBufs& operator=(const DevBufs&) = delete;
    ~DevBufs() { for (void* p : ptrs) gl_dev_free(ctx, p); }
    template <class T> T* alloc(size_t n) {
        void* p = nullptr;
        glck(ctx, gl_dev_alloc(ctx, (int64_t)std::max<size_t>(n * sizeof(T), 16), &p), "gl_dev_alloc");
        ptrs.push_back(p);
        return static_cast<T*>(p);
    }
    template <class T> T* upload(const T* h, size_t n) {
        T* d = alloc<T>(n);
        if (n) glck(ctx, gl_memcpy_h2d(ctx, d, h, (int64_t)(n * sizeof(T))), "gl_memcpy_h2d");
        return d;
    }
};

// Where kept reference q's tiles of sample k lie in the cohort depths: off/len at [q * S + k] (ref.ID() indexes the index's
// reference array, indexcov.go:656).  len is 0 when the sample lacks the reference or its median is 0 (indexcov.go:140-142);
// such an empty slice starts at the sample's first tile.  longest[q] is over every sample, so the table needs every median.
struct IcSlices {
    std::vector<int64_t> off, len, longest;
};

static IcSlices ic_slices(const std::vector<const IcRef*>& kept, const std::vector<std::vector<int64_t>>& size_ptr,
                          const std::vector<int64_t>& sample_ptr, const std::vector<double>& med) {
    const size_t S = med.size();
    IcSlices sl;
    sl.off.resize(kept.size() * S); sl.len.assign(kept.size() * S, 0); sl.longest.assign(kept.size(), 0);
    for (size_t q = 0; q < kept.size(); q++) {
        const int id = kept[q]->id;
        for (size_t k = 0; k < S; k++) {
            const size_t j = q * S + k;
            sl.off[j] = sample_ptr[k];
            if (id + 1 >= (int)size_ptr[k].size() || med[k] == 0) continue;
            sl.off[j] += size_ptr[k][id];
            sl.len[j] = size_ptr[k][id + 1] - size_ptr[k][id];
            sl.longest[q] = std::max(sl.longest[q], sl.len[j]);
        }
    }
    return sl;
}

// -n (I7, indexcov.go:670-672): the values of each kept non-sex reference are normalised across the samples as one
// S x longest matrix and written back into their slices of dep.  Each reference id is normalised once, so a reference that
// -c lists twice shows the same values both times, as the reference's fresh NormalizedDepth slices do (indexcov.go:129-151).
static void ic_extranorm(gl_ctx* ctx, const std::vector<const IcRef*>& kept, const std::vector<std::string>& sexes_wanted,
                         const IcSlices& sl, size_t S, float* dep) {
    std::vector<float> mat;
    std::vector<int32_t> lens(S);
    for (size_t q = 0; q < kept.size(); q++) {
        const size_t longest = (size_t)sl.longest[q];
        const int id = kept[q]->id;
        if (longest == 0 || same_chrom(sexes_wanted, kept[q]->name) ||
            std::any_of(kept.begin(), kept.begin() + (long)q, [&](const IcRef* r) { return r->id == id; }))
            continue;
        const int64_t* off = &sl.off[q * S];
        mat.assign(S * longest, 0.f);
        for (size_t k = 0; k < S; k++) {
            lens[k] = (int32_t)sl.len[q * S + k];
            memcpy(&mat[k * longest], dep + off[k], (size_t)lens[k] * 4);
        }
        glck(ctx, gl_indexcov_xnorm(ctx, mat.data(), lens.data(), (int32_t)S, (int32_t)longest), "gl_indexcov_xnorm");
        for (size_t k = 0; k < S; k++) memcpy(dep + off[k], &mat[k * longest], (size_t)lens[k] * 4);
    }
}

// Phase B on one GPU, over the resident depths d_dep of samples [a, b), which begin at cohort tile t0: the "%.3g" token of
// every value (I6) into tok_all, and the slot histograms + counters (I4+I5) of every (sample, kept reference) pair into
// counts_all / b4_all at [k * nq + q].  That order keeps one GPU's samples together, so each array comes home in one copy.
static void ic_tokens_counts(gl_ctx* c, const float* d_dep, size_t a, size_t b, const std::vector<int64_t>& sample_ptr,
                             const IcSlices& sl, uint8_t* tok_all, int32_t* counts_all, int64_t* b4_all) {
    const size_t S = sample_ptr.size() - 1, nq = sl.longest.size(), nseg = nq * (b - a);
    const int64_t t0 = sample_ptr[a], tiles = sample_ptr[b] - t0;
    DevBufs tmp(c);
    if (tiles) {
        uint8_t* d_tok = tmp.alloc<uint8_t>((size_t)tiles * 10);
        glck(c, gl_format_g3_device(c, d_dep, tiles, d_tok), "gl_format_g3_device");
        glck(c, gl_memcpy_d2h(c, tok_all + (size_t)t0 * 10, d_tok, tiles * 10), "gl_memcpy_d2h");
    }
    if (nseg == 0) return;
    std::vector<int64_t> seg_start(nseg), seg_len(nseg), seg_longest(nseg);
    for (size_t k = a; k < b; k++)
        for (size_t q = 0; q < nq; q++) {
            const size_t j = (k - a) * nq + q;
            seg_start[j] = sl.off[q * S + k] - t0;
            seg_len[j] = sl.len[q * S + k];
            seg_longest[j] = sl.longest[q];
        }
    const int64_t* d_ss = tmp.upload(seg_start.data(), nseg);
    const int64_t* d_sl = tmp.upload(seg_len.data(), nseg);
    const int64_t* d_lg = tmp.upload(seg_longest.data(), nseg);
    int32_t* d_c = tmp.alloc<int32_t>(nseg * GL_INDEXCOV_SLOTS);
    int64_t* d_b = tmp.alloc<int64_t>(nseg * 4);
    glck(c, gl_indexcov_counts_segs_device(c, d_dep, d_ss, d_sl, d_lg, (int32_t)nseg, d_c, d_b), "gl_indexcov_counts_segs_device");
    glck(c, gl_memcpy_d2h(c, counts_all + a * nq * GL_INDEXCOV_SLOTS, d_c, (int64_t)nseg * GL_INDEXCOV_SLOTS * 4), "gl_memcpy_d2h");
    glck(c, gl_memcpy_d2h(c, b4_all + a * nq * 4, d_b, (int64_t)nseg * 32), "gl_memcpy_d2h");
}

// ---- the depth and ROC charts (plot.cu, DESIGN §1.14).  Chart c shows kept reference q_of[c]; dataset (c, k) is sample
// k's line, drawn with index k + 1, so the last sample lies on top as in the reference (plot.go:142-144 + asPng:480-481).
struct IcPlots {
    std::vector<size_t> q_of;
    std::vector<int64_t> sel;          // gl_plot_select's {first, m, stride} of dataset (c, k) at [(c * S + k) * 3]
    std::vector<float> yext;           // ... and its y extent at [(c * S + k) * 2]
    std::vector<double> xf;            // per chart: gl_plot_transform of the extent over every sample
    std::vector<double> ext;           // per chart: that extent, {xmin, xmax, ymin, ymax}
};

// The extent of chart c over every drawn dataset (gonum's DataRange over the plotted vertices); mult scales the index.
static void ic_plot_extent(IcPlots& pl, size_t c, size_t S, double mult) {
    double e[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
    for (size_t k = 0; k < S; k++) {
        const int64_t* s3 = &pl.sel[(c * S + k) * 3];
        if (s3[1] == 0) continue;
        e[0] = std::min(e[0], (double)s3[0] * mult);
        e[1] = std::max(e[1], (double)(s3[0] + (s3[1] - 1) * s3[2]) * mult);
        e[2] = std::min(e[2], (double)pl.yext[(c * S + k) * 2]);
        e[3] = std::max(e[3], (double)pl.yext[(c * S + k) * 2 + 1]);
    }
    if (e[0] > e[1]) e[0] = e[1] = e[2] = e[3] = 0;                       // nothing drawn
    pl.ext.insert(pl.ext.end(), e, e + 4);
    double xf[4];
    if (gl_plot_transform(e, GL_PLOT_W, GL_PLOT_H, xf) != GL_OK) fatal(1, "gl_plot_transform failed");
    pl.xf.insert(pl.xf.end(), xf, xf + 4);
}

// The datasets of samples [a, b) on the GPU holding them from cohort tile t0: off / len inside d_dep, in (c, k) order.
static void ic_plot_slices(const IcPlots& pl, const IcSlices& sl, size_t S, size_t a, size_t b, int64_t t0, std::vector<int64_t>& off,
                           std::vector<int64_t>& len) {
    off.clear(); len.clear();
    for (size_t c = 0; c < pl.q_of.size(); c++)
        for (size_t k = a; k < b; k++) {
            off.push_back(sl.off[pl.q_of[c] * S + k] - t0);
            len.push_back(sl.len[pl.q_of[c] * S + k]);
        }
}

// round 1 on one GPU: the selection of its samples' datasets, into pl.sel / pl.yext
static void ic_plot_select(gl_ctx* c, const float* d_dep, size_t a, size_t b, const std::vector<int64_t>& sample_ptr, const IcSlices& sl,
                           IcPlots& pl) {
    const size_t S = sample_ptr.size() - 1, nk = b - a, n = pl.q_of.size() * nk;
    if (n == 0) return;
    std::vector<int64_t> off, len, sel(n * 3);
    std::vector<float> yext(n * 2);
    ic_plot_slices(pl, sl, S, a, b, sample_ptr[a], off, len);
    DevBufs tmp(c);
    int64_t* d_sel = tmp.alloc<int64_t>(n * 3);
    float* d_y = tmp.alloc<float>(n * 2);
    glck(c, gl_plot_select_device(c, d_dep, tmp.upload(off.data(), n), tmp.upload(len.data(), n), (int32_t)n, d_sel, d_y), "gl_plot_select_device");
    glck(c, gl_memcpy_d2h(c, sel.data(), d_sel, (int64_t)n * 24), "gl_memcpy_d2h");
    glck(c, gl_memcpy_d2h(c, yext.data(), d_y, (int64_t)n * 8), "gl_memcpy_d2h");
    for (size_t j = 0; j < n; j++) {
        const size_t g = (j / nk) * S + a + j % nk;
        std::copy(&sel[j * 3], &sel[j * 3 + 3], &pl.sel[g * 3]);
        std::copy(&yext[j * 2], &yext[j * 2 + 2], &pl.yext[g * 2]);
    }
}

// The path text of a vector chart (INDEXCOV_FMT; plot.cu): dataset j's bytes are text[pos[j] .. pos[j + 1]).
struct IcPathText {
    std::vector<int64_t> pos;
    std::vector<char> text;
};

// gl_plot_path_*_size, the lengths home, then gl_plot_path_*_emit into a buffer of exactly that size and the text home
template <class Size, class Emit>
static void ic_path_text(gl_ctx* c, DevBufs& tmp, size_t n, const Size& size, const Emit& emit, IcPathText& pt) {
    int64_t* d_len = tmp.alloc<int64_t>(n);
    int64_t* d_pos = tmp.alloc<int64_t>(n + 1);
    glck(c, size(d_len, d_pos), "gl_plot_path_*_size");
    pt.pos.resize(n + 1);
    glck(c, gl_memcpy_d2h(c, pt.pos.data(), d_pos, (int64_t)(n + 1) * 8), "gl_memcpy_d2h");
    const int64_t total = pt.pos[n];
    pt.text.resize((size_t)total);
    char* d_txt = tmp.alloc<char>((size_t)total);
    glck(c, emit(d_pos, total, d_txt), "gl_plot_path_*_emit");
    glck(c, gl_memcpy_d2h(c, pt.text.data(), d_txt, total), "gl_memcpy_d2h");
}

// round 2 on one GPU: the index images of its samples' lines, with the cohort's extents (img: every chart), and with
// vfmt >= 0 their depth charts' path text in (chart, sample) order
static void ic_plot_raster(gl_ctx* c, const float* d_dep, size_t a, size_t b, const std::vector<int64_t>& sample_ptr, const IcSlices& sl,
                           const IcPlots& pl, double r, uint32_t* img, int vfmt, IcPathText& pt) {
    const size_t S = sample_ptr.size() - 1, nk = b - a, nc = pl.q_of.size(), n = nc * nk;
    std::vector<int64_t> off, len, sel(n * 3);
    std::vector<int32_t> chart(n);
    std::vector<uint32_t> draw(n);
    ic_plot_slices(pl, sl, S, a, b, sample_ptr[a], off, len);
    for (size_t j = 0; j < n; j++) {
        const size_t k = a + j % nk, ch = j / nk;
        std::copy(&pl.sel[(ch * S + k) * 3], &pl.sel[(ch * S + k) * 3 + 3], &sel[j * 3]);
        chart[j] = (int32_t)ch; draw[j] = (uint32_t)(k + 1);
    }
    DevBufs tmp(c);
    const int64_t* d_off = tmp.upload(off.data(), n);
    const int64_t* d_sel = tmp.upload(sel.data(), n * 3);
    const int32_t* d_chart = tmp.upload(chart.data(), n);
    const double* d_xf = tmp.upload(pl.xf.data(), nc * 4);
    uint32_t* d_img = tmp.alloc<uint32_t>(nc * GL_PLOT_W * GL_PLOT_H);
    glck(c, gl_plot_raster_series_device(c, d_dep, d_off, d_sel, (double)GL_TILE_WIDTH, d_chart, tmp.upload(draw.data(), n), (int32_t)n, d_xf,
                                         (int32_t)nc, GL_PLOT_W, GL_PLOT_H, r, d_img), "gl_plot_raster_series_device");
    glck(c, gl_memcpy_d2h(c, img, d_img, (int64_t)(nc * GL_PLOT_W * GL_PLOT_H * 4)), "gl_memcpy_d2h");
    if (vfmt < 0) return;
    ic_path_text(c, tmp, n,
                 [&](int64_t* d_len, int64_t* d_pos) {
                     return gl_plot_path_series_size(c, d_dep, d_off, d_sel, (double)GL_TILE_WIDTH, d_chart, (int32_t)n, d_xf, (int32_t)nc,
                                                     GL_PLOT_DEPTH, vfmt, d_len, d_pos);
                 },
                 [&](const int64_t* d_pos, int64_t total, char* d_txt) {
                     return gl_plot_path_series_emit(c, d_dep, d_off, d_sel, (double)GL_TILE_WIDTH, d_chart, (int32_t)n, d_xf, (int32_t)nc,
                                                     GL_PLOT_DEPTH, vfmt, d_pos, total, d_txt, total);
                 },
                 pt);
}

// the path text of explicit vertices (the ROC and sex charts), on GPU 0 as their rasters are
static void ic_path_text_xy(gl_ctx* c, const std::vector<double>& x, const std::vector<double>& y, const std::vector<int64_t>& ptr,
                            const std::vector<int32_t>& chart, const double* xf, size_t n_charts, int kind, int vfmt, IcPathText& pt) {
    const size_t n = chart.size();
    DevBufs tmp(c);
    const double* d_x = tmp.upload(x.data(), x.size());
    const double* d_y = tmp.upload(y.data(), y.size());
    const int64_t* d_ptr = tmp.upload(ptr.data(), ptr.size());
    const int32_t* d_chart = tmp.upload(chart.data(), n);
    const double* d_xf = tmp.upload(xf, n_charts * 4);
    ic_path_text(c, tmp, n,
                 [&](int64_t* d_len, int64_t* d_pos) {
                     return gl_plot_path_xy_size(c, d_x, d_y, d_ptr, d_chart, (int32_t)n, d_xf, (int32_t)n_charts, kind, vfmt, d_len, d_pos);
                 },
                 [&](const int64_t* d_pos, int64_t total, char* d_txt) {
                     return gl_plot_path_xy_emit(c, d_x, d_y, d_ptr, d_chart, (int32_t)n, d_xf, (int32_t)n_charts, kind, vfmt, d_pos, total,
                                                 d_txt, total);
                 },
                 pt);
}

// One vector chart file: its datasets' path text (data[d], len[d]) in draw order, each stroked in rgb[3 d ..].
struct IcVecFile {
    std::string path, xtitle, ytitle;
    int kind = GL_PLOT_DEPTH;
    double ext[4] = {0, 0, 0, 0};
    double width = 0.8;
    std::vector<uint8_t> rgb;
    std::vector<const char*> data;
    std::vector<int64_t> len;
};

// The vector charts (INDEXCOV_FMT): the files and the path text they point into.  vfmt < 0: none.
struct IcVectors {
    int vfmt = -1;
    std::string ext;                                       // "svg" or "eps"
    std::vector<IcPathText> depth;                         // per GPU: its samples' depth paths, in (chart, sample) order
    IcPathText roc, sex;
    std::vector<IcVecFile> files;
    std::string file_of(const std::string& png) const { return png.substr(0, png.size() - 3) + ext; }   // plot.go:533-534
};

// every vector chart file, one pool task each
static void ic_vectors_write(const IcVectors& vec) {
    glhost::ThreadPool::global().run((int64_t)vec.files.size(), [&](int64_t t, int) {
        const IcVecFile& f = vec.files[(size_t)t];
        if (gl_plot_vector_write(f.path.c_str(), f.kind, vec.vfmt, f.ext, f.xtitle.c_str(), f.ytitle.c_str(), (int32_t)f.data.size(), f.rgb.data(),
                                 f.width, f.data.data(), f.len.data()) != GL_OK)
            fatal(1, "%s", gl_last_error(nullptr));
    });
}

static void ic_write_png(const std::string& path, const uint32_t* img, const std::vector<uint8_t>& palette, int kind, const double* ext,
                         const std::string& xtitle, const std::string& ytitle) {
    std::vector<uint8_t> rgb((size_t)GL_PLOT_CW * GL_PLOT_CH * 3);
    if (gl_plot_compose(img, palette.data(), (int32_t)(palette.size() / 3), kind, ext, xtitle.c_str(), ytitle.c_str(), rgb.data()) != GL_OK)
        fatal(1, "gl_plot_compose: %s", gl_last_error(nullptr));
    int64_t n = 0;
    gl_plot_png(rgb.data(), GL_PLOT_CW, GL_PLOT_CH, nullptr, 0, &n);
    std::vector<uint8_t> png((size_t)n);
    if (gl_plot_png(rgb.data(), GL_PLOT_CW, GL_PLOT_CH, png.data(), n, &n) != GL_OK) fatal(1, "gl_plot_png: %s", gl_last_error(nullptr));
    FILE* f = fopen(path.c_str(), "wb");
    if (!f || fwrite(png.data(), 1, (size_t)n, f) != (size_t)n || fclose(f) != 0) fatal(1, "cannot write %s", path.c_str());
}

// The ROC charts (their lines rasterised on GPU 0 from host vertex arrays), every chart's PNG on the host pool, and
// index.html.  INDEXCOV_N_BACKGROUNDS=n greys the first n samples in every chart (plot.go:87-101).
// what the pages show besides the depth and ROC lines
struct IcReport {
    const std::vector<std::string>& names;
    const float* dep;                                        // the cohort depths (after -n) at the slices of sl
    const IcSlices& sl;
    const std::map<std::string, std::vector<double>>& sexes;
    const std::vector<uint64_t>& mapped, & unmapped;
    const std::vector<int64_t>& bins;                        // per sample: out, lo, hi, in
    const std::vector<double>& pcs;                          // S x 5
    int32_t n_pc;
    const double* vars;                                      // n_pc variance-explained fractions
};

// tooltip titles: names[dataset][point]
static std::string ic_tooltip(const std::vector<std::vector<std::string>>& names) {
    std::string js = "  var names = [";
    for (size_t d = 0; d < names.size(); d++) {
        js += d ? ",[" : "[";
        for (size_t i = 0; i < names[d].size(); i++) js += (i ? "," : "") + glhtml::quote(names[d][i]);
        js += "]";
    }
    return js + "];\n  chart.options.tooltips.callbacks.title = function(tts, data) {\n    var out = [];\n"
                "    tts.forEach(function(ti) { out.push(names[ti.datasetIndex][ti.index]); });\n    return out.join(\",\");\n  };";
}

// asValues (plot.go:66-83) of n values at v, every vertex: x = i * mult, y = min(v, 2.5)
static void ic_as_values(const float* v, size_t n, double mult, glhtml::Dataset& ds) {
    size_t i = 0;
    while (i < n && v[i] == 0.f) i++;
    for (; i < n; i++) { ds.x.push_back((double)i * mult); ds.y.push_back((double)(v[i] > 2.5f ? 2.5f : v[i])); }
}

static void ic_write_text(const std::string& path, const std::string& text) {
    FILE* f = fopen(path.c_str(), "w");
    if (!f || fwrite(text.data(), 1, text.size(), f) != text.size() || fclose(f) != 0) fatal(1, "cannot write %s", path.c_str());
}

// With INDEXCOV_FMT, vec gets the list of vector chart files: the depth paths were made in phase B (vec.depth, one entry per
// GPU, whose samples are [cut[g], cut[g + 1])); the ROC and sex paths are made here on GPU 0.
static void ic_plots_write(gl_ctx* ctx, const std::string& base, const std::string& dir, const std::vector<const IcRef*>& kept,
                           const IcPlots& pl, const std::vector<std::vector<float>>& roc_vals, const std::vector<uint32_t>& depth_img,
                           double r, size_t S, const IcReport& rep, const std::vector<size_t>& cut, IcVectors& vec) {
    const size_t kMaxSamples = 100;                                         // indexcov.go:528 maxSamples
    if (S > kMaxSamples)
        fprintf(stderr, "indexcov: creating only static (no interactive) plots for depth because # of samples %zu is > %zu\n", S, kMaxSamples);
    int32_t n_bg = 0;
    if (const char* v = getenv("INDEXCOV_N_BACKGROUNDS")) {
        char* end = nullptr;
        const long n = strtol(v, &end, 10);
        if (*v && end && !*end) {
            n_bg = (int32_t)std::max(-1L, std::min(n, (long)INT32_MAX));
            fprintf(stderr, "[indexcov] setting first %d samples as background\n", n_bg);
        }
    }
    std::vector<uint8_t> palette(3 * (S + 1), 255);                         // palette[v] for draw index v; 0 stays white
    for (size_t k = 0; k < S; k++) gl_plot_color((int32_t)k, n_bg, &palette[3 * (k + 1)]);
    const size_t nc = pl.q_of.size(), img_n = (size_t)GL_PLOT_W * GL_PLOT_H;
    const double roc_mult = (1.0 / (double)GL_INDEXCOV_SLOTS) / (2.0 / 3.0);   // plot.go:336, x = i * (1/70) / (2/3)
    IcPlots rp;
    rp.q_of = pl.q_of;
    rp.sel.resize(nc * S * 3); rp.yext.resize(nc * S * 2);
    std::vector<double> x, y;
    std::vector<int64_t> ptr(1, 0);
    std::vector<int32_t> chart;
    std::vector<uint32_t> draw;
    std::vector<int64_t> off(S), len(S, GL_INDEXCOV_SLOTS);
    for (size_t k = 0; k < S; k++) off[k] = (int64_t)k * GL_INDEXCOV_SLOTS;
    for (size_t c = 0; c < nc; c++) {
        const float* v = roc_vals[c].data();
        if (roc_vals[c].size() != S * GL_INDEXCOV_SLOTS) fatal(1, "indexcov: no ROC values for chart %zu", c);
        gl_plot_select_host(v, off.data(), len.data(), (int32_t)S, &rp.sel[c * S * 3], &rp.yext[c * S * 2]);
        ic_plot_extent(rp, c, S, roc_mult);
        for (size_t k = 0; k < S; k++) {
            const int64_t* s3 = &rp.sel[(c * S + k) * 3];
            if (s3[1] < 2) continue;
            for (int64_t j = 0; j < s3[1]; j++) {
                const int64_t i = s3[0] + j * s3[2];
                const float f = v[k * GL_INDEXCOV_SLOTS + (size_t)i];
                x.push_back((double)i * roc_mult);
                y.push_back((double)(f > 2.5f ? 2.5f : f));
            }
            ptr.push_back((int64_t)x.size()); chart.push_back((int32_t)c); draw.push_back((uint32_t)(k + 1));
        }
    }
    std::vector<uint32_t> roc_img(nc * img_n);
    if (nc) glck(ctx, gl_plot_raster_xy(ctx, x.data(), y.data(), ptr.data(), chart.data(), draw.data(), (int32_t)chart.size(), rp.xf.data(),
                                        (int32_t)nc, GL_PLOT_W, GL_PLOT_H, r, roc_img.data()), "gl_plot_raster_xy");
    if (vec.vfmt >= 0) {
        if (nc) ic_path_text_xy(ctx, x, y, ptr, chart, rp.xf.data(), nc, GL_PLOT_PLAIN, vec.vfmt, vec.roc);
        const double w = gl_plot_line_width((int32_t)S);
        for (size_t c = 0; c < nc; c++) {                                   // asPng's vector copies (plot.go:527-536)
            const std::string& chrom = kept[pl.q_of[c]]->name;
            IcVecFile d, o;
            d.path = vec.file_of(base + "-depth-" + chrom + ".png"); d.kind = GL_PLOT_DEPTH; std::copy(&pl.ext[c * 4], &pl.ext[c * 4 + 4], d.ext);
            d.xtitle = "position on " + chrom; d.ytitle = "scaled coverage"; d.width = w;
            for (size_t g = 0; g + 1 < cut.size(); g++) {
                const size_t nk = cut[g + 1] - cut[g];
                for (size_t k = cut[g]; k < cut[g + 1]; k++) {
                    const size_t j = c * nk + (k - cut[g]);
                    const IcPathText& pt = vec.depth[g];
                    d.data.push_back(pt.text.data() + pt.pos[j]); d.len.push_back(pt.pos[j + 1] - pt.pos[j]);
                    d.rgb.insert(d.rgb.end(), &palette[3 * (k + 1)], &palette[3 * (k + 1)] + 3);
                }
            }
            o.path = vec.file_of(base + "-roc-" + chrom + ".png"); o.kind = GL_PLOT_PLAIN; std::copy(&rp.ext[c * 4], &rp.ext[c * 4 + 4], o.ext);
            o.xtitle = "scaled coverage for " + chrom; o.ytitle = "proportion of regions covered"; o.width = w;
            for (size_t i = 0; i < chart.size(); i++) {
                if ((size_t)chart[i] != c) continue;
                o.data.push_back(vec.roc.text.data() + vec.roc.pos[i]); o.len.push_back(vec.roc.pos[i + 1] - vec.roc.pos[i]);
                o.rgb.insert(o.rgb.end(), &palette[3 * draw[i]], &palette[3 * draw[i]] + 3);
            }
            vec.files.push_back(std::move(d));
            vec.files.push_back(std::move(o));
        }
    }
    const std::string stem = base.substr(base.find_last_of('/') + 1);
    const std::string back = "<p><a href=\"index.html\">back to index</a></p>\n";
    glhost::ThreadPool::global().run((int64_t)(4 * nc), [&](int64_t t, int) {
        const size_t c = (size_t)t / 4;
        const std::string& chrom = kept[pl.q_of[c]]->name;
        if (t % 4 == 2) {                                                   // plotDepths' page (plot.go:110-164), S <= 100 only
            if (S > kMaxSamples) return;
            glhtml::Chart ch;
            ch.name = "depth"; ch.xlabel = "position on " + chrom; ch.ylabel = "scaled coverage";
            const double w = S > 50 ? 0.2 : (S > 30 ? 0.3 : 0.4);
            for (size_t kk = S; kk-- > 0;) {                                // the reference adds the datasets last sample first
                glhtml::Dataset ds;
                ds.label = rep.names[kk]; ds.xfmt = "%.0f"; ds.width = w;
                gl_plot_color((int32_t)kk, n_bg, ds.rgb);
                const size_t j = pl.q_of[c] * S + kk;
                ic_as_values(rep.dep + rep.sl.off[j], (size_t)rep.sl.len[j], (double)GL_TILE_WIDTH, ds);
                ch.data.push_back(std::move(ds));
            }
            ic_write_text(base + "-depth-" + chrom + ".html", glhtml::page("indexcov depth " + chrom, back + glhtml::chart_html(ch, 850, 550)));
            return;
        }
        if (t % 4 == 3) {                                                   // plotROCs' page (plot.go:318-353)
            glhtml::Chart ch;
            ch.name = "roc"; ch.xlabel = "scaled coverage for " + chrom; ch.ylabel = "proportion of regions covered";
            for (size_t kk = S; kk-- > 0;) {
                glhtml::Dataset ds;
                ds.label = (int64_t)kk < n_bg ? "background" : rep.names[kk]; ds.width = 2;
                gl_plot_color((int32_t)kk, n_bg, ds.rgb);
                ic_as_values(&roc_vals[c][kk * GL_INDEXCOV_SLOTS], GL_INDEXCOV_SLOTS, roc_mult, ds);
                ch.data.push_back(std::move(ds));
            }
            ic_write_text(base + "-roc-" + chrom + ".html", glhtml::page("indexcov roc " + chrom, back + glhtml::chart_html(ch, 850, 550)));
            return;
        }
        if (t % 4 == 0)
            ic_write_png(base + "-depth-" + chrom + ".png", &depth_img[c * img_n], palette, GL_PLOT_DEPTH, &pl.ext[c * 4], "position on " + chrom,
                         "scaled coverage");
        else
            ic_write_png(base + "-roc-" + chrom + ".png", &roc_img[c * img_n], palette, GL_PLOT_PLAIN, &rp.ext[c * 4],
                         "scaled coverage for " + chrom, "proportion of regions covered");
    });
    // ---- index.html (indexcov.go:896-953): the cohort charts, then every chromosome's images
    std::string body = "<h3>indexcov: " + std::to_string(S) + " samples</h3>\n<p><a href=\"" + stem + ".ped\">" + stem + ".ped</a> | <a href=\"" +
                       stem + ".bed.gz\">" + stem + ".bed.gz</a> | <a href=\"" + stem + ".roc\">" + stem + ".roc</a></p>\n";
    const uint8_t green[3] = {110, 250, 59}, grey[3] = {180, 180, 180};
    auto scatter = [&](glhtml::Dataset& ds, const uint8_t* rgb, const char* label) {
        ds.line = false; ds.width = 4; ds.label = label; std::copy(rgb, rgb + 3, ds.rgb);
    };
    if (rep.sexes.size() >= 2) {                                            // plotSex (plot.go:412-474) + its PNG (indexcov.go:918-921)
        auto it = rep.sexes.begin();
        const std::string k0 = it->first, k1 = std::next(it)->first;
        const std::vector<double>& cn0 = it->second;
        const std::vector<double>& cn1 = std::next(it)->second;
        std::vector<int> inferred(S);
        std::set<int> cns;
        for (size_t k = 0; k < S; k++) { inferred[k] = (int)(0.5 + cn0[k]); cns.insert(inferred[k]); }
        glhtml::Chart ch;
        ch.name = "sex"; ch.xlabel = k0 + " Copy Number"; ch.ylabel = k1 + " Copy Number"; ch.legend = true;
        std::vector<std::vector<std::string>> tips;
        std::vector<double> sx, sy;
        std::vector<int64_t> sptr(1, 0);
        std::vector<int32_t> schart;
        std::vector<uint32_t> sdraw;
        std::vector<uint8_t> spal(3, 255);
        double e[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
        for (int cn : cns) {                                                 // ascending inferred CN
            glhtml::Dataset ds;
            scatter(ds, green, "");
            ds.label = "Inferred CN for " + k0 + ": " + std::to_string(cn); ds.width = 6;
            gl_plot_color(cn, 0, ds.rgb);
            tips.emplace_back();
            for (size_t k = (size_t)std::max<int32_t>(n_bg, 0); k < S; k++) {
                if (inferred[k] != cn) continue;
                ds.x.push_back(cn0[k]); ds.y.push_back(cn1[k]); tips.back().push_back(rep.names[k]);
                e[0] = std::min(e[0], cn0[k]); e[1] = std::max(e[1], cn0[k]); e[2] = std::min(e[2], cn1[k]); e[3] = std::max(e[3], cn1[k]);
            }
            sx.insert(sx.end(), ds.x.begin(), ds.x.end()); sy.insert(sy.end(), ds.y.begin(), ds.y.end());
            sptr.push_back((int64_t)sx.size()); schart.push_back(0); sdraw.push_back((uint32_t)(sdraw.size() + 1));
            spal.insert(spal.end(), ds.rgb, ds.rgb + 3);
            ch.data.push_back(std::move(ds));
        }
        ch.tooltip_js = "  chart.options.hover.mode = 'index';\n" + ic_tooltip(tips);
        body += "<h4>sex</h4>\n" + glhtml::chart_html(ch, 550, 550);
        if (!(e[0] <= e[1])) e[0] = e[1] = e[2] = e[3] = 0;
        // asPng draws the scatter as lines joining each dataset's points in sample order
        double xf[4];
        std::vector<uint32_t> simg((size_t)GL_PLOT_SQ_W * GL_PLOT_SQ_H);
        if (gl_plot_transform(e, GL_PLOT_SQ_W, GL_PLOT_SQ_H, xf) != GL_OK) fatal(1, "gl_plot_transform failed");
        glck(ctx, gl_plot_raster_xy(ctx, sx.data(), sy.data(), sptr.data(), schart.data(), sdraw.data(), (int32_t)schart.size(), xf, 1,
                                    GL_PLOT_SQ_W, GL_PLOT_SQ_H, gl_plot_line_radius((int32_t)schart.size()), simg.data()), "gl_plot_raster_xy");
        std::vector<uint8_t> rgb((size_t)GL_PLOT_SQ_CW * GL_PLOT_SQ_CH * 3);
        if (gl_plot_compose(simg.data(), spal.data(), (int32_t)(spal.size() / 3), GL_PLOT_SQUARE, e, (k0 + " Copy Number").c_str(),
                            (k1 + " Copy Number").c_str(), rgb.data()) != GL_OK)
            fatal(1, "gl_plot_compose: %s", gl_last_error(nullptr));
        int64_t n = 0;
        gl_plot_png(rgb.data(), GL_PLOT_SQ_CW, GL_PLOT_SQ_CH, nullptr, 0, &n);
        std::vector<uint8_t> png((size_t)n);
        if (gl_plot_png(rgb.data(), GL_PLOT_SQ_CW, GL_PLOT_SQ_CH, png.data(), n, &n) != GL_OK) fatal(1, "gl_plot_png failed");
        ic_write_text(base + "-sex.png", std::string(png.begin(), png.begin() + n));
        if (vec.vfmt >= 0) {
            ic_path_text_xy(ctx, sx, sy, sptr, schart, xf, 1, GL_PLOT_SQUARE, vec.vfmt, vec.sex);
            IcVecFile f;
            f.path = vec.file_of(base + "-sex.png"); f.kind = GL_PLOT_SQUARE; std::copy(e, e + 4, f.ext);
            f.xtitle = k0 + " Copy Number"; f.ytitle = k1 + " Copy Number"; f.width = gl_plot_line_width((int32_t)schart.size());
            for (size_t i = 0; i < schart.size(); i++) {
                f.data.push_back(vec.sex.text.data() + vec.sex.pos[i]); f.len.push_back(vec.sex.pos[i + 1] - vec.sex.pos[i]);
            }
            f.rgb.assign(spal.begin() + 3, spal.end());
            vec.files.push_back(std::move(f));
        }
        body += "<p><img src=\"" + stem + "-sex.png\" alt=\"sex\"></p>\n";
    }
    std::vector<std::string> fg_names;
    for (size_t k = (size_t)std::max<int32_t>(n_bg, 0); k < S; k++) fg_names.push_back(rep.names[k]);
    bool anygt = false;
    for (size_t k = 0; k < S; k++) if (rep.mapped[k] || rep.unmapped[k]) anygt = true;
    if (anygt) {                                                            // plotMapped (plot.go:355-410)
        glhtml::Chart ch;
        ch.name = "mapped"; ch.xlabel = "log(mapped reads)"; ch.ylabel = "log(unmapped reads)";
        glhtml::Dataset ds;
        scatter(ds, green, "samples");
        for (size_t k = (size_t)std::max<int32_t>(n_bg, 0); k < S; k++) {
            ds.x.push_back(log1p((double)rep.mapped[k])); ds.y.push_back(log1p((double)rep.unmapped[k]));
        }
        ch.data.push_back(std::move(ds));
        ch.tooltip_js = "  chart.options.hover.mode = 'index';\n" + ic_tooltip({fg_names});
        body += "<h4>mapped and unmapped reads</h4>\n" + glhtml::chart_html(ch, 550, 550);
    }
    std::vector<std::string> bg_names((size_t)std::min<int64_t>(std::max<int32_t>(n_bg, 0), (int64_t)S), "background");
    auto two_sets = [&](glhtml::Chart& ch, const std::function<void(size_t, double&, double&)>& xy, const char* xf, const char* yf) {
        glhtml::Dataset bg, fg;
        scatter(bg, grey, "samples"); scatter(fg, green, "samples");
        bg.xfmt = fg.xfmt = xf; bg.yfmt = fg.yfmt = yf;
        for (size_t k = 0; k < S; k++) {
            double x, y;
            xy(k, x, y);
            glhtml::Dataset& d = (int64_t)k < n_bg ? bg : fg;
            d.x.push_back(x); d.y.push_back(y);
        }
        std::vector<std::vector<std::string>> tips;
        if (n_bg > 0) { ch.data.push_back(std::move(bg)); tips.push_back(bg_names); }
        ch.data.push_back(std::move(fg)); tips.push_back(fg_names);
        ch.tooltip_js = ic_tooltip(tips);
    };
    {                                                                       // plotBins (plot.go:166-249)
        glhtml::Chart ch;
        ch.name = "bins"; ch.xlabel = "proportion of bins with depth < 0.15"; ch.ylabel = "proportion of bins with depth outside of (0.85, 1.15)";
        two_sets(ch, [&](size_t k, double& x, double& y) {
            const double tot = (double)(rep.bins[k * 4 + 3] + rep.bins[k * 4 + 0]);
            x = (double)rep.bins[k * 4 + 1] / std::max(tot, 1.0);
            y = (double)rep.bins[k * 4 + 0] / tot;
        }, "%.5f", "%.3f");
        body += "<h4>bins</h4>\n" + glhtml::chart_html(ch, 550, 550);
    }
    if (rep.n_pc >= 3)                                                      // plotPCA (plot.go:251-316)
        for (int pc : {2, 3}) {
            glhtml::Chart ch;
            ch.name = "pca" + std::to_string(pc);
            char lx[96], ly[96];
            snprintf(lx, sizeof lx, "PC1 (variance explained: %.2f%%)", 100 * rep.vars[0]);
            snprintf(ly, sizeof ly, "PC%d (variance explained: %.2f%%)", pc, 100 * rep.vars[pc - 1]);
            ch.xlabel = lx; ch.ylabel = ly;
            two_sets(ch, [&](size_t k, double& x, double& y) { x = rep.pcs[k * 5]; y = rep.pcs[k * 5 + (size_t)pc - 1]; }, "%.2f", "%.2f");
            ch.tooltip_js = "  chart.options.hover.mode = 'index';\n" + ch.tooltip_js;
            body += "<h4>PCA: PC1 vs PC" + std::to_string(pc) + "</h4>\n" + glhtml::chart_html(ch, 550, 550);
        }
    for (size_t c = 0; c < nc; c++) {
        const std::string& chrom = kept[pl.q_of[c]]->name;
        const std::string dimg = "<img src=\"" + stem + "-depth-" + chrom + ".png\" alt=\"depth " + chrom + "\">";
        body += "<div><h4>" + chrom + "</h4><a href=\"" + stem + "-roc-" + chrom + ".html\"><img src=\"" + stem + "-roc-" + chrom +
                ".png\" alt=\"roc " + chrom + "\"></a> " +
                (S <= kMaxSamples ? "<a href=\"" + stem + "-depth-" + chrom + ".html\">" + dimg + "</a>" : dimg) + "</div>\n";
    }
    const std::string index_path = dir + "/index.html";
    ic_write_text(index_path, glhtml::page("indexcov", body));
    fprintf(stderr, "indexcov finished: see %s for overview of output\n", index_path.c_str());   // indexcov.go:454
}

// .ped (indexcov.go:815-894)
static void ic_write_ped(const std::string& base, const std::vector<std::string>& names, const std::map<std::string, std::vector<double>>& sexes,
                         const std::vector<int64_t>& bins, const std::vector<float>& slopes, const std::vector<double>& pcs, int32_t n_pc,
                         const std::vector<uint64_t>& mapped, const std::vector<uint64_t>& unmapped) {
    const size_t S = names.size();
    FILE* ped = fopen((base + ".ped").c_str(), "w");
    if (!ped) fatal(1, "cannot create %s.ped", base.c_str());
    bool anygt = false;
    for (size_t k = 0; k < S; k++) if (mapped[k] > 0 || unmapped[k] > 0) anygt = true;
    fprintf(ped, "#family_id\tsample_id\tpaternal_id\tmaternal_id\tsex\tphenotype");
    for (auto& kv : sexes) fprintf(ped, "\tCN%s", kv.first.c_str());
    fprintf(ped, "\tbins.out\tbins.lo\tbins.hi\tbins.in\tslope\tp.out");
    for (int j = 0; j < n_pc; j++) fprintf(ped, "\tPC%d", j + 1);
    if (anygt) fprintf(ped, "\tmapped\tunmapped");
    fputc('\n', ped);
    for (size_t k = 0; k < S; k++) {
        const int inferred = sexes.empty() ? -9 : (int)(0.5 + sexes.begin()->second[k]);
        fprintf(ped, "unknown\t%s\t-9\t-9\t%d\t-9", names[k].c_str(), inferred);
        for (auto& kv : sexes) fprintf(ped, "\t%s", go_float("%.2f", kv.second[k]).c_str());
        fprintf(ped, "\t%lld\t%lld\t%lld\t%lld\t%s\t%s", (long long)bins[k * 4 + 0], (long long)bins[k * 4 + 1], (long long)bins[k * 4 + 2],
                (long long)bins[k * 4 + 3], go_float("%.3f", (double)slopes[k]).c_str(),
                go_float("%.2f", (double)bins[k * 4 + 0] / (double)bins[k * 4 + 3]).c_str());
        for (int j = 0; j < n_pc; j++) fprintf(ped, "\t%s", go_float("%.2f", pcs[k * 5 + (size_t)j]).c_str());
        if (anygt) fprintf(ped, "\t%llu\t%llu", (unsigned long long)mapped[k], (unsigned long long)unmapped[k]);
        fputc('\n', ped);
    }
    fclose(ped);
}

static int cmd_indexcov(int argc, char** argv) {
    std::string dir, exclude = "^chrEBV$|^NC|_random$|Un_|^HLA\\-|_alt$|hap\\d$", sex = "X,Y", chrom, fai, gpus = "0";
    bool includegl = false, extranorm = false;
    ArgParser ap;
    ap.prog = "goleft indexcov";
    ap.add("directory", 'd', &dir, true); ap.addb("includegl", 'e', &includegl); ap.add("excludepatt", 0, &exclude);
    ap.add("sex", 'X', &sex); ap.add("chrom", 'c', &chrom); ap.add("fai", 'f', &fai); ap.addb("extranormalize", 'n', &extranorm);
    ap.add("gpus", 0, &gpus);                       // extension: GPUs to use (0 = every visible one); samples are sharded over them
    bool noplots = false;
    ap.addb("noplots", 0, &noplots);                // extension: no charts; index.html only lists the outputs
    ap.parse(argc, argv);
    // INDEXCOV_FMT (plot.go:527-536): every chart PNG gets a vector copy, X.svg for "svg" and X.eps for any other non-empty value
    IcVectors vec;
    if (const char* v = getenv("INDEXCOV_FMT"))
        if (*v && !noplots) { vec.ext = strcmp(v, "svg") == 0 ? "svg" : "eps"; vec.vfmt = vec.ext == "svg" ? GL_PLOT_SVG : GL_PLOT_EPS; }
    std::vector<std::string> bams = ap.positional;
    if (bams.empty()) ap.fail("bam is required");
    std::vector<std::string> sexes_wanted;
    { size_t p = 0; for (;;) { size_t c = sex.find(',', p); std::string t = sex.substr(p, c == std::string::npos ? std::string::npos : c - p); if (!t.empty()) sexes_wanted.push_back(t); if (c == std::string::npos) break; p = c + 1; } }
    std::regex excl(exclude);
    mkdir(dir.c_str(), 0755);

    // references (indexcov.go:344-374): BAM header of the first input, or the .fai
    std::vector<IcRef> refs;
    if (ends_with(bams[0], ".bam")) {
        glhts::BamHeader h;
        std::string e = glhts::bam_read_header(bams[0], h);
        if (!e.empty()) fatal(1, "%s", e.c_str());
        for (size_t i = 0; i < h.refs.size(); i++) refs.push_back({h.refs[i].name, h.refs[i].length, (int)i});
        if (!chrom.empty()) {                                               // RefsFromBam appends the named chrom (:336-338)
            std::string c = chrom.compare(0, 3, "chr") == 0 ? chrom.substr(3) : chrom;
            bool found = false;
            for (size_t i = 0; i < h.refs.size() && !found; i++) {
                const std::string& n = h.refs[i].name;
                if (c == n || (n.compare(0, 3, "chr") == 0 && c == n.substr(3))) { refs.push_back({n, h.refs[i].length, (int)i}); found = true; }
            }
            if (!found) fatal(1, "indexcov: chromosome: %s not found", chrom.c_str());
        }
    } else if (!fai.empty()) {
        std::vector<glhts::RefInfo> r;
        std::string e = glhts::fai_read(fai, r);
        if (!e.empty()) fatal(1, "error opening fai: %s. Is is present?", fai.c_str());
        for (auto& x : r) if (chrom.empty() || x.name == chrom) refs.push_back({x.name, x.length, (int)refs.size()});
        if (refs.empty()) fatal(1, "ERROR: didn't find any usable chromosomes in %s", fai.c_str());
    } else {
        fatal(1, "indexcov: since no .fai was specified, expected input to be a list of bams");
    }

    // indexes (indexcov.go:471-525)
    const bool ic_timing = getenv("GL_TIMING") != nullptr;               // phase wall clocks on stderr
    double ic_t0 = now_s(), ic_tp = ic_t0;
    auto ic_mark = [&](const char* what) { if (ic_timing) { const double t = now_s(); fprintf(stderr, "[indexcov timing] %-28s %.3f s\n", what, t - ic_tp); ic_tp = t; } };
    const size_t S = bams.size();
    std::vector<std::string> names(S);
    std::vector<glhts::BaiIndex> idx(S);
    std::vector<std::vector<glhts::CraiSlices>> crai(S);
    // the reference reads the indexes on 8 goroutines (indexcov.go:417-434); here every pool thread takes files.  The first
    // error in INPUT order is the one reported, whatever thread met it.
    std::vector<std::string> read_err(S);
    glhost::ThreadPool::global().run((int64_t)S, [&](int64_t ii, int) {
        const size_t i = (size_t)ii;
        const std::string& b = bams[i];
        if (ends_with(b, ".crai")) {                                       // indexcov.go:474-496
            read_err[i] = glhts::crai_read(b, crai[i]);
            names[i] = short_name(b, true, nullptr);
            return;
        }
        read_err[i] = glhts::bai_read(bai_path(b), idx[i]);
        if (!read_err[i].empty()) return;
        if (ends_with(b, ".bai") || ends_with(b, ".csi")) names[i] = short_name(b, true, nullptr);
        else { glhts::BamHeader h; read_err[i] = glhts::bam_read_header(b, h); if (read_err[i].empty()) names[i] = short_name(b, false, &h); }
    });
    for (size_t i = 0; i < S; i++) {
        if (!read_err[i].empty()) fatal(1, "%s", read_err[i].c_str());
        if (!ends_with(bams[i], ".crai")) refuse_wide_csi(idx[i], bai_path(bams[i]), "indexcov");
    }

    ic_mark("read indexes");
    // ---- GPUs (SURVEY 8(e): samples are independent through I5 -> sample-sharded over the GPUs; the rows need every sample
    //      of a tile, and they are assembled on the host, so the "gather" is each GPU's D2H into its slice of the cohort arrays)
    const GpuPlan gp = resolve_gpus(gpus, S, "goleft indexcov");
    const int G = gp.G;
    fprintf(stderr, "indexcov: running on %zu indexes\n", bams.size());

    // ---- I1 for the whole cohort (indexcov/types.go:45-82): every sample's linear-index offsets go up once, one descriptor per
    //      (sample, reference with >= 2 entries); CRAM samples bring host-made pseudo-tile sizes
    std::vector<int64_t> sample_ptr(1, 0);
    std::vector<std::vector<int64_t>> size_ptr(S);                          // per sample: CSR over its refs
    std::vector<uint64_t> mapped(S, 0), unmapped(S, 0);
    std::vector<uint64_t> voff_all;
    std::vector<int64_t> desc_voff, desc_size;
    std::vector<int32_t> desc_n;
    std::vector<size_t> desc_begin(S + 1, 0), voff_begin(S + 1, 0);         // per sample: its first descriptor / first offset
    std::vector<std::vector<int64_t>> crai_tiles(S);                        // CRAM samples: the sizes themselves
    for (size_t i = 0; i < S; i++) {
        const int64_t base = sample_ptr.back();
        desc_begin[i] = desc_n.size(); voff_begin[i] = voff_all.size();
        if (ends_with(bams[i], ".crai")) {                                  // CRAM: interpolated pseudo-tiles
            crai_sizes(crai[i], crai_tiles[i], size_ptr[i]);
            if (size_ptr[i].back() < 1) fatal(1, "indexcov: no usable chromsomes in bam: %s", bams[i].c_str());
            sample_ptr.push_back(base + size_ptr[i].back());
            continue;
        }
        const size_t nr = idx[i].ioffsets.size();
        std::vector<int64_t> sp(nr + 1, 0);
        for (size_t r = 0; r < nr; r++) {
            const std::vector<uint64_t>& io = idx[i].ioffsets[r];
            mapped[i] += idx[i].mapped[r]; unmapped[i] += idx[i].unmapped[r];
            sp[r + 1] = sp[r] + (io.size() >= 2 ? (int64_t)io.size() - 1 : 0);          // types.go:68-72
            if (io.size() >= 2) {
                desc_voff.push_back((int64_t)voff_all.size()); desc_n.push_back((int32_t)io.size()); desc_size.push_back(base + sp[r]);
                voff_all.insert(voff_all.end(), io.begin(), io.end());
            }
        }
        if (sp[nr] < 1) fatal(1, "indexcov: no usable chromsomes in bam: %s", bams[i].c_str());   // indexcov.go:100-102
        sample_ptr.push_back(base + sp[nr]);
        size_ptr[i] = sp;
    }
    desc_begin[S] = desc_n.size(); voff_begin[S] = voff_all.size();
    const int64_t total = sample_ptr.back();
    // contiguous sample ranges with about total/G tiles each
    std::vector<size_t> cut((size_t)G + 1, S);
    cut[0] = 0;
    for (int g = 1; g < G; g++) {
        const int64_t want = total / G * g;
        cut[(size_t)g] = (size_t)(std::lower_bound(sample_ptr.begin(), sample_ptr.end(), want) - sample_ptr.begin());
        cut[(size_t)g] = std::min(std::max(cut[(size_t)g], cut[(size_t)g - 1]), S);
    }

    const std::string base = dir + "/" + dir.substr(dir.find_last_of('/') == std::string::npos ? 0 : dir.find_last_of('/') + 1) + "-indexcov";
    // the references that are reported (exclude pattern, indexcov.go:637-646)
    std::vector<const IcRef*> kept;
    {
        int n_reported = 0;
        for (const IcRef& ref : refs) {
            if (!exclude.empty() && std::regex_search(ref.name, excl)) {
                if (n_reported < 10) { fprintf(stderr, "indexcv: excluding chromosome: %s because of exclude-pattern: %s\n", ref.name.c_str(), exclude.c_str()); if (++n_reported == 10) fprintf(stderr, "not reporting further skipped chromosomes\n"); }
                continue;
            }
            kept.push_back(&ref);
        }
    }
    // cohort-sized arrays that the GPUs overwrite completely: not zero-filled (a std::vector's constructor page-faulted through
    // 0.8 GB on one thread: 0.6 s of the 313-sample run)
    std::vector<double> med(S);
    const size_t nq = kept.size();
    RawBuf<float> dep; dep.resize((size_t)total);
    RawBuf<uint8_t> tok_all; tok_all.resize((size_t)total * 10 + 16);
    RawBuf<int32_t> counts_all; counts_all.resize(S * nq * GL_INDEXCOV_SLOTS);
    RawBuf<int64_t> b4_all; b4_all.resize(S * nq * 4);

    std::vector<gl_ctx*> ctxs((size_t)G, nullptr);
    // phase A (per GPU, its samples): I1 + I2 + I3 on the device, medians + depths home; the depths stay resident for phase B
    struct Shard { DevBufs resident; float* d_dep = nullptr; };
    std::vector<Shard> shard((size_t)G);
    // a single GPU's work runs on this thread: on a worker thread the row assembly below, which reads what the D2H copies
    // wrote, took about 0.3 s longer for 313 samples
    auto run_on_gpus = [&](const std::function<void(int)>& fn) {
        if (G == 1) fn(0);
        else for (std::thread& t : start_workers(gp, fn)) t.join();
    };
    ic_mark("host arrays");
    std::vector<std::array<double, 4>> gpu_t((size_t)G);                     // per GPU: ctx, upload + I1, I2 + I3, D2H
    run_on_gpus([&](int g) {
        double tg0 = now_s();
        gl_ctx* c = open_ctx(g % gp.n_dev, "goleft indexcov");
        ctxs[(size_t)g] = c;
        gpu_t[(size_t)g] = {now_s() - tg0, 0, 0, 0};
        tg0 = now_s();
        const size_t a = cut[(size_t)g], b = cut[(size_t)g + 1];
        const int64_t t0 = sample_ptr[a], tiles = sample_ptr[b] - t0;
        Shard& sd = shard[(size_t)g];
        sd.resident.ctx = c;
        if (b == a) return;
        DevBufs tmp(c);
        int64_t* d_sizes = tmp.alloc<int64_t>((size_t)tiles);
        const size_t d0 = desc_begin[a], d1 = desc_begin[b], v0 = voff_begin[a], v1 = voff_begin[b];
        if (d1 > d0) {
            std::vector<int64_t> dv(desc_voff.begin() + (long)d0, desc_voff.begin() + (long)d1), ds(desc_size.begin() + (long)d0, desc_size.begin() + (long)d1);
            for (auto& x : dv) x -= (int64_t)v0;
            for (auto& x : ds) x -= t0;
            DevBufs in(c);
            const uint64_t* d_voff = in.upload(voff_all.data() + v0, v1 - v0);
            const int64_t* d_dv = in.upload(dv.data(), dv.size());
            const int32_t* d_dn = in.upload(desc_n.data() + d0, d1 - d0);
            const int64_t* d_ds = in.upload(ds.data(), ds.size());
            const int rc = gl_indexcov_sizes_batch_device(c, d_voff, d_dv, d_dn, d_ds, (int64_t)(d1 - d0), d_sizes);
            if (rc == GL_ERANGE) fatal(2, "panic: expected positive change in vOffset");                 // types.go:75-77
            glck(c, rc, "gl_indexcov_sizes_batch_device");
        }
        for (size_t i = a; i < b; i++)
            if (!crai_tiles[i].empty())
                glck(c, gl_memcpy_h2d(c, d_sizes + (sample_ptr[i] - t0), crai_tiles[i].data(), (int64_t)crai_tiles[i].size() * 8), "gl_memcpy_h2d");
        glck(c, gl_sync(c), "gl_sync");
        gpu_t[(size_t)g][1] = now_s() - tg0; tg0 = now_s();
        // I2+I3 for the shard in one kernel, on the resident sizes (indexcov.go:83-151)
        std::vector<int64_t> sp(sample_ptr.begin() + (long)a, sample_ptr.begin() + (long)b + 1);
        for (auto& x : sp) x -= t0;
        const int64_t* d_sp = tmp.upload(sp.data(), sp.size());
        double* d_med = tmp.alloc<double>(b - a);
        sd.d_dep = sd.resident.alloc<float>((size_t)tiles);
        glck(c, gl_indexcov_cohort_device(c, d_sizes, d_sp, (int32_t)(b - a), d_med, sd.d_dep), "gl_indexcov_cohort_device");
        glck(c, gl_sync(c), "gl_sync");
        gpu_t[(size_t)g][2] = now_s() - tg0; tg0 = now_s();
        glck(c, gl_memcpy_d2h(c, med.data() + a, d_med, (int64_t)(b - a) * 8), "gl_memcpy_d2h");
        glck(c, gl_memcpy_d2h(c, dep.data() + t0, sd.d_dep, tiles * 4), "gl_memcpy_d2h");
        gpu_t[(size_t)g][3] = now_s() - tg0;
    });
    std::vector<uint64_t>().swap(voff_all);
    if (ic_timing)
        for (int g = 0; g < G; g++)
            fprintf(stderr, "[indexcov timing]   gpu %d: gl_ctx_create %.3f s, upload + I1 %.3f s, I2 + I3 %.3f s, D2H %.3f s\n", g, gpu_t[(size_t)g][0],
                    gpu_t[(size_t)g][1], gpu_t[(size_t)g][2], gpu_t[(size_t)g][3]);
    ic_mark("I1 + I2 + I3 (GPU, + D2H)");

    glhts::BgzfWriter bgz(base + ".bed.gz");
    FILE* roc = fopen((base + ".roc").c_str(), "w");
    if (!bgz.ok() || !roc) fatal(1, "cannot create outputs in %s", dir.c_str());
    { std::string h = "#chrom\tstart\tend"; for (auto& n : names) h += "\t" + n; h += "\n"; bgz.write(h.data(), h.size()); }

    // `longest` of a reference is over all samples (and needs every median), hence the barrier between the phases
    const IcSlices sl = ic_slices(kept, size_ptr, sample_ptr, med);
    gl_ctx* ctx = ctxs[0];                                                  // -n and the PCA run on GPU 0
    if (extranorm) {                                                        // -n rewrites the values; each GPU takes its range back
        ic_extranorm(ctx, kept, sexes_wanted, sl, S, dep.data());
        run_on_gpus([&](int g) {
            const int64_t t0 = sample_ptr[cut[(size_t)g]], tiles = sample_ptr[cut[(size_t)g + 1]] - t0;
            if (tiles) glck(ctxs[(size_t)g], gl_memcpy_h2d(ctxs[(size_t)g], shard[(size_t)g].d_dep, dep.data() + t0, tiles * 4), "gl_memcpy_h2d");
        });
        ic_mark("-n (GPU 0, + H2D)");
    }
    // ---- phase B: the values no longer change, so every token and count comes from two launches per GPU
    // the charts (indexcov.go:707-726): every kept reference with more than 2 tiles, GL* ones only with -e
    IcPlots pl;
    if (!noplots)
        for (size_t q = 0; q < nq; q++)
            if ((includegl || kept[q]->name.compare(0, 2, "GL") != 0) && sl.longest[q] > 2) pl.q_of.push_back(q);
    const size_t n_charts = pl.q_of.size();
    pl.sel.assign(n_charts * S * 3, 0); pl.yext.assign(n_charts * S * 2, 0);
    run_on_gpus([&](int g) {
        const size_t a = cut[(size_t)g], b = cut[(size_t)g + 1];
        if (b == a) return;
        ic_tokens_counts(ctxs[(size_t)g], shard[(size_t)g].d_dep, a, b, sample_ptr, sl, tok_all.data(), counts_all.data(), b4_all.data());
        ic_plot_select(ctxs[(size_t)g], shard[(size_t)g].d_dep, a, b, sample_ptr, sl, pl);
    });
    // depth charts: the extents over every sample, then each GPU draws its samples' lines and the images combine by max
    const size_t img_n = (size_t)GL_PLOT_W * GL_PLOT_H;
    const double plot_r = gl_plot_line_radius((int32_t)S);
    std::vector<uint32_t> depth_img;
    if (n_charts) {
        for (size_t c = 0; c < n_charts; c++) ic_plot_extent(pl, c, S, (double)GL_TILE_WIDTH);
        std::vector<std::vector<uint32_t>> part((size_t)G);
        vec.depth.resize((size_t)G);
        run_on_gpus([&](int g) {
            const size_t a = cut[(size_t)g], b = cut[(size_t)g + 1];
            if (b == a) return;
            part[(size_t)g].resize(n_charts * img_n);
            ic_plot_raster(ctxs[(size_t)g], shard[(size_t)g].d_dep, a, b, sample_ptr, sl, pl, plot_r, part[(size_t)g].data(), vec.vfmt,
                           vec.depth[(size_t)g]);
        });
        depth_img.assign(n_charts * img_n, 0);
        for (auto& p : part)
            for (size_t i = 0; i < p.size(); i++) depth_img[i] = std::max(depth_img[i], p[i]);
    }
    shard.clear();                                                          // frees the resident depths
    for (int g = 1; g < G; g++) gl_ctx_destroy(ctxs[(size_t)g]);
    ic_mark("tokens + counts (GPU, + D2H)");

    std::map<std::string, std::vector<double>> sexes;
    std::vector<int64_t> bins(S * 4, 0);
    std::vector<float> slopes(S, 0);
    int n_slopes = 0;
    // the PCA's byte matrix (indexcov.go:686-705): every kept reference that is not a sex chromosome gives each sample
    // longest + 1 columns, its clipped values' bytes and then zeros (the range loop leaves i at the last index, or -1)
    std::vector<std::vector<float>> roc_vals(n_charts);                     // the ROC values (S x 70) of each chart's reference
    std::vector<int64_t> pca_col(nq, -1);
    int64_t pca_D = 0;
    for (size_t q = 0; q < nq; q++)
        if (!same_chrom(sexes_wanted, kept[q]->name)) { pca_col[q] = pca_D; pca_D += sl.longest[q] + 1; }
    const int64_t pca_rank = std::min<int64_t>((int64_t)S, pca_D);          // gonum's min(S, D) components
    const int64_t pca_ld = (pca_D + 63) / 64 * 64;
    RawBuf<uint8_t> pca_x;
    if (pca_rank >= 3) pca_x.resize(S * (size_t)pca_ld);
    for (size_t q = 0; q < nq; q++) {
        const IcRef& ref = *kept[q];
        const size_t longest = (size_t)sl.longest[q];
        const int64_t* off = &sl.off[q * S];
        const int64_t* lens = &sl.len[q * S];
        const bool is_sex = same_chrom(sexes_wanted, ref.name);
        // bed.gz rows (indexcov.go:678-680,1038-1048): every "%.3g" comes from the GPU formatter as a 10-byte token; the rows
        // are put together by all host threads, 256 rows per task, and handed to the BGZF writer in order
        {
            const size_t kRows = 256, n_tasks = (longest + kRows - 1) / kRows;
            std::vector<std::string> parts(n_tasks);
            glhost::ThreadPool::global().run((int64_t)n_tasks, [&](int64_t t, int) {
                std::string& out = parts[(size_t)t];
                out.reserve(kRows * (ref.name.size() + 24 + S * 7));
                char num[48];
                const size_t i0 = (size_t)t * kRows, i1 = std::min(longest, i0 + kRows);
                for (size_t i = i0; i < i1; i++) {
                    out += ref.name;
                    out.append(num, (size_t)snprintf(num, sizeof num, "\t%zu\t%zu", i * 16384, (i + 1) * 16384));
                    for (size_t k = 0; k < S; k++) {
                        out.push_back('\t');
                        if (i >= (size_t)lens[k]) { out.push_back('0'); continue; }
                        const size_t t = (size_t)off[k] + i;
                        const uint8_t* tk = &tok_all[t * 10];
                        if (tk[9]) out.append(reinterpret_cast<const char*>(tk), tk[9]);
                        else out += go_float("%.3g", (double)dep[t]);                               // magnitude outside the kernel's range
                    }
                    out.push_back('\n');
                }
            });
            for (const std::string& part : parts) bgz.write(part.data(), part.size());
        }
        if (is_sex) {
            if (longest > 0) { std::vector<double> cn(S); for (size_t k = 0; k < S; k++) cn[k] = get_cn(&dep[(size_t)off[k]], (size_t)lens[k]); sexes[ref.name] = cn; }
        } else {
            for (size_t k = 0; k < S; k++)
                for (size_t j = 0; j < 4; j++) bins[k * 4 + j] += b4_all[(k * nq + q) * 4 + j];
            if (pca_rank >= 3)
                glhost::ThreadPool::global().run((int64_t)S, [&](int64_t k, int) {
                    uint8_t* row = &pca_x[(size_t)k * (size_t)pca_ld + (size_t)pca_col[q]];
                    const size_t n = (size_t)lens[k];
                    for (size_t i = 0; i < n; i++) row[i] = glpca::pca8_byte(dep[(size_t)off[k] + i]);
                    memset(row + n, 0, longest + 1 - n);
                });
        }
        if (longest > 0) {                                                  // writeROCs (indexcov.go:1018-1036)
            std::string h = "#chrom\tcov"; for (auto& n : names) h += "\t" + n; h += "\n";
            fputs(h.c_str(), roc);
            std::vector<float> rocs(S * GL_INDEXCOV_SLOTS);
            for (size_t k = 0; k < S; k++) {
                int tot[GL_INDEXCOV_SLOTS];
                const int32_t* c = &counts_all[(k * nq + q) * GL_INDEXCOV_SLOTS];
                tot[GL_INDEXCOV_SLOTS - 1] = c[GL_INDEXCOV_SLOTS - 1];
                for (int i = GL_INDEXCOV_SLOTS - 2; i >= 0; i--) tot[i] = tot[i + 1] + c[i];
                const float mx = (float)tot[0];
                for (int i = 0; i < GL_INDEXCOV_SLOTS; i++) rocs[k * GL_INDEXCOV_SLOTS + i] = (float)tot[i] / mx;
            }
            for (size_t c = 0; c < n_charts; c++) if (pl.q_of[c] == q) roc_vals[c] = rocs;
            for (int i = 0; i < GL_INDEXCOV_SLOTS; i++) {
                fprintf(roc, "%s\t%.2f", ref.name.c_str(), (double)i / (70.0 * (2.0 / 3.0)));
                for (size_t k = 0; k < S; k++) fprintf(roc, "\t%s", go_float("%.2f", (double)rocs[k * GL_INDEXCOV_SLOTS + i]).c_str());
                fputc('\n', roc);
            }
            if ((includegl || ref.name.compare(0, 2, "GL") != 0) && longest > 2 && !is_sex && longest > 100) {
                const double sm = 2.0 / 3.0;                                // updateSlopes (indexcov.go:739-750)
                const int ilo = (int)(0.5 + (sm - 0.1) * 70), ihi = (int)(0.5 + (sm + 0.1) * 70);
                const float scalar = (float)ref.len / 1e6f;
                for (size_t k = 0; k < S; k++) slopes[k] += (rocs[k * 70 + ilo] - rocs[k * 70 + ihi]) * scalar;
                n_slopes++;
            }
        }
    }
    ic_mark("rows + roc per reference");
    bgz.close();
    fclose(roc);
    ic_mark("bgzf close");
    for (size_t k = 0; k < S; k++) slopes[k] = slopes[k] / (float)n_slopes;
    if (sexes.size() != sexes_wanted.size()) {                              // checkSexes (indexcov.go:760-770)
        std::string keys; for (auto& kv : sexes) keys += (keys.empty() ? "" : ",") + kv.first;
        if (sexes.empty() && sex != "X,Y") fatal(1, "(FATAL) indexcov: expected %zu sex chromosomes, found: %zu.", sexes_wanted.size(), sexes.size());
        fprintf(stderr, "(WARNING) indexcov: expected %zu sex chromosomes, found: %zu.\nyou can set the expected with --sex '%s'\n", sexes_wanted.size(), sexes.size(), keys.c_str());
    }
    // pca (indexcov.go:773-807): the first five components on GPU 0, once every reference's bytes are in; fewer than five
    // components are logged, and fewer than three give no PC columns.  Without any kept autosome (D = 0) the reference's
    // gonum panics on the empty matrix; here that is 0 components (DESIGN §1.11).
    if (sexes.empty()) fprintf(stderr, "sex chromosomes not found.\n");
    int32_t n_pc = 0;
    std::vector<double> pcs;
    double sv[5] = {0, 0, 0, 0, 0}, vars[5] = {0, 0, 0, 0, 0};
    if (pca_rank < 5) fprintf(stderr, "got: %lld principal components\n", (long long)pca_rank);
    if (pca_rank < 3) {
        fprintf(stderr, "indexcov: %lld principal components, not plotting\n", (long long)pca_rank);
    } else {
        pcs.resize(S * 5);
        glck(ctx, gl_indexcov_pca(ctx, pca_x.data(), pca_ld, (int32_t)S, pca_D, 5, pcs.data(), sv, &n_pc, nullptr), "gl_indexcov_pca");
        double total = 0;                                                   // the PCA labels' vars: s_k^2 / ||X_c||_F^2
        if (!noplots && gl_indexcov_pca_total(pca_x.data(), pca_ld, (int32_t)S, pca_D, &total) != GL_OK) fatal(1, "gl_indexcov_pca_total failed");
        for (int j = 0; j < n_pc; j++) vars[j] = total > 0 ? sv[j] * sv[j] / total : 0;
    }
    ic_mark("pca");
    ic_write_ped(base, names, sexes, bins, slopes, pcs, n_pc, mapped, unmapped);
    if (!noplots) {
        ic_plots_write(ctx, base, dir, kept, pl, roc_vals, depth_img, plot_r, S,
                       IcReport{names, dep.data(), sl, sexes, mapped, unmapped, bins, pcs, n_pc, vars}, cut, vec);
        ic_mark("charts");
        if (vec.vfmt >= 0) {
            ic_vectors_write(vec);
            ic_mark("vector");
        }
    } else {                                                                // --noplots: a plain list of the outputs
        const std::string index_path = dir + "/index.html";
        FILE* ih = fopen(index_path.c_str(), "w");
        if (ih) {
            const std::string stem = base.substr(base.find_last_of('/') + 1);
            fprintf(ih, "<html><head><title>indexcov</title></head><body><p>goleft_b200 indexcov: %zu samples; plots are not built by this engine.</p><ul>"
                        "<li><a href=\"%s.bed.gz\">%s.bed.gz</a></li><li><a href=\"%s.roc\">%s.roc</a></li><li><a href=\"%s.ped\">%s.ped</a></li></ul></body></html>\n",
                    S, stem.c_str(), stem.c_str(), stem.c_str(), stem.c_str(), stem.c_str(), stem.c_str());
            fclose(ih);
            fprintf(stderr, "indexcov finished: see %s for overview of output\n", index_path.c_str());   // indexcov.go:454
        }
    }
    gl_ctx_destroy(ctx);
    if (ic_timing) fprintf(stderr, "[indexcov timing] %-28s %.3f s\n", "total", now_s() - ic_t0);
    return 0;
}

// ------------------------------------------------------------------------------------------------ covstats
// V1 + V2 (covstats.go:122-220): gl_bam_covstats samples the records and computes the reference's Stats on the device;
// a file it cannot take (GL_ESTATE), or GL_GPU_FEED=0, goes through gl_bam_covstats_host, with the same tail.
//
// --gpus N: the BAMs go through a BamQueue, dealt dynamically (a BAM the device refuses costs several times more on the host
// route).  A worker starts reading the first batch of the BAM it opened ahead (gl_bam_covstats_prefetch) as soon as the
// current one's sampling call has consumed its own prefetch, so that the read overlaps the rest of the current BAM's work
// (the --hist tail, the .bai read for the mapped counts, the commit).  The main thread prints the rows as they commit.
struct CsJob : BamJob {
    gl_covstats st;
    std::vector<double> H;
    std::string names, not_found;
    long long genome = 0;
    unsigned long long mapped = 0;
};

static int cmd_covstats(int argc, char** argv) {
    // the header is printed before the arguments are parsed (covstats.go:224-226)
    printf("coverage\tinsert_mean\tinsert_sd\tinsert_5th\tinsert_95th\ttemplate_mean\ttemplate_sd\tpct_unmapped\tpct_bad_reads\tpct_duplicate\tpct_proper_pair\tread_length\tbam\tsample\n");
    std::string nstr = "1000000", regions, fasta, hist, gpus = "0";
    ArgParser ap;
    ap.prog = "goleft covstats";
    ap.add("n", 'n', &nstr); ap.add("regions", 'r', &regions); ap.add("fasta", 'f', &fasta); ap.add("hist", 0, &hist);
    ap.add("gpus", 0, &gpus);                       // extension: GPUs to use (0 = every visible one); the BAMs are dealt to them
    ap.parse(argc, argv);
    if (ap.positional.empty()) ap.fail("bams is required");
    const int N = atoi(nstr.c_str());
    const int kSkip = 100000;
    const std::vector<std::string>& bams = ap.positional;
    const size_t S = bams.size();
    const GpuPlan gp = resolve_gpus(gpus, S, "goleft covstats");
    BamQueue<CsJob> queue(bams);
    // BAM i on worker context c: everything but the output
    auto run = [&](gl_ctx* c, size_t i, gl_bam* ahead) {
        CsJob& J = queue.jobs[i];
        const std::string& bam = bams[i];
        gl_bam* bh = J.bh;
        gl_covstats& st = J.st;
        auto sample = [&](bool device) {
            int rc = device ? gl_bam_covstats(c, bh, N, kSkip, &st, nullptr, 0) : gl_bam_covstats_host(c, bh, N, kSkip, &st, nullptr, 0);
            if (rc == GL_ERANGE && st.h_len > 0 && !hist.empty()) {              // H is wanted: the tail over the samples this call left
                const int32_t *rl = nullptr, *ins = nullptr, *tm = nullptr;
                std::vector<int32_t> v;
                if (device) {
                    const int32_t *d_rl = nullptr, *d_ins = nullptr, *d_tm = nullptr;
                    if ((rc = gl_bam_covstats_samples(c, &d_rl, &d_ins, &d_tm)) != GL_OK) return rc;
                    v.resize((size_t)(st.n_read_len + 2 * st.n_insert));
                    if (st.n_read_len && (rc = gl_memcpy_d2h(c, v.data(), d_rl, st.n_read_len * 4)) != GL_OK) return rc;
                    if (st.n_insert && ((rc = gl_memcpy_d2h(c, v.data() + st.n_read_len, d_ins, st.n_insert * 4)) != GL_OK ||
                                        (rc = gl_memcpy_d2h(c, v.data() + st.n_read_len + st.n_insert, d_tm, st.n_insert * 4)) != GL_OK)) return rc;
                    rl = v.data(); ins = rl + st.n_read_len; tm = ins + st.n_insert;
                } else if ((rc = gl_bam_covstats_host_samples(bh, &rl, &ins, &tm)) != GL_OK) return rc;
                gl_covstats t = st;
                J.H.resize((size_t)st.h_len);
                rc = gl_covstats_tail(c, rl, st.n_read_len, ins, st.n_insert, tm, st.n_insert, &t, J.H.data(), st.h_len);
            } else if (rc == GL_ERANGE && st.h_len > 0) rc = GL_OK;              // the row does not print H
            return rc;
        };
        int rc = SegSource::gpu_feed() ? sample(true) : GL_ESTATE;
        if (rc == GL_ESTATE) rc = sample(false);
        // a prefetch that cannot start (no pinned memory) leaves the read to the call, which reports its own failures
        if (ahead && SegSource::gpu_feed()) (void)gl_bam_covstats_prefetch(c, ahead, N, kSkip);
        if (rc == GL_EINVAL && st.n_insert > 0 && st.n_insert < 3) { J.code = 2; J.msg = "panic: runtime error: index out of range (covstats madFilter needs at least 3 insert sizes)"; return; }
        if (rc == GL_ERANGE) { J.code = 2; J.msg = std::string("panic: runtime error: makeslice: len out of range (") + gl_last_error(c) + ")"; return; }
        if (rc != GL_OK) { J.code = 1; J.msg = gl_last_error(c); return; }
        const glhts::BamHeader& hdr = bh->f.header;
        for (auto& s : hdr.sample_names()) J.names += (J.names.empty() ? "" : ",") + s;
        if (J.names.empty()) J.names = "<no-read-groups>";
        glhts::BaiIndex bai;
        bool have_idx = false;
        if (ends_with(bam, ".bam")) {
            std::string be = glhts::bai_read(bai_path(bam), bai);
            if (!be.empty()) { J.code = 1; J.msg = be; return; }
            have_idx = true;
        }
        for (size_t r = 0; r < hdr.refs.size(); r++) {                              // covstats.go:256-267
            J.genome += hdr.refs[r].length;
            if (have_idx) {
                if (r >= bai.has_stats.size() || !bai.has_stats[r]) {
                    if (hdr.refs[r].name.find("random") == std::string::npos && hdr.refs[r].length > 10000) J.not_found += (J.not_found.empty() ? "" : ",") + hdr.refs[r].name;
                    continue;
                }
                J.mapped += bai.mapped[r];
            }
        }
    };
    queue.start(gp, [&](int g, std::string& err) {
        gl_ctx* c = nullptr;
        if (gl_ctx_create(g % gp.n_dev, &c) != GL_OK) err = std::string("goleft covstats: ") + gl_last_error(nullptr);
        return c;
    }, run, [](gl_ctx* c) { gl_ctx_destroy(c); });
    // the commit: rows in argument order
    long long region_genome = -1;
    for (size_t i = 0; i < S; i++) {
        const CsJob& J = queue.wait(i);
        if (J.code) { queue.stop(); fatal(J.code, "%s", J.msg.c_str()); }
        const std::string& bam = bams[i];
        const gl_covstats& st = J.st;
        const double pBad = st.proportion_bad, pDup = st.proportion_duplicate, pProper = st.proportion_properly_paired, pUnmapped = st.proportion_unmapped;
        const double rlMean = st.read_length_mean, insMean = st.insert_mean, insSd = st.insert_sd, tMean = st.template_mean, tSd = st.template_sd;
        const int pct5 = st.insert_pct5, pct95 = st.insert_pct95, maxRead = st.max_read_length;
        if (!hist.empty()) {                                                        // Stats.H (covstats.go:202-217), one line per entry
            const std::string hp = hist + "." + J.names + ".template_hist.tsv";
            FILE* hf = fopen(hp.c_str(), "w");
            if (!hf) { const int e = errno; queue.stop(); fatal(1, "open %s: %s", hp.c_str(), strerror(e)); }
            for (size_t j = 0; j < J.H.size(); j++) fprintf(hf, "%lld\t%s\n", (long long)maxRead + (long long)j, go_float("%.6g", J.H[j]).c_str());
            fclose(hf);
        }
        if (!J.not_found.empty()) fprintf(stderr, "chromosomes: %s not found in %s\n", J.not_found.c_str(), bam.c_str());
        long long genome = J.genome;
        if (!regions.empty()) {                                                     // covstats.go:36-55, read once
            if (region_genome < 0) {
                gzFile f = gzopen(regions.c_str(), "rb");
                if (!f) queue.stop();                                               // read_lines ends the run with the open error
                else gzclose(f);
                region_genome = 0;
                for (const std::string& ln : read_lines(regions, true)) {
                    size_t t1 = ln.find('\t');
                    if (t1 == std::string::npos) continue;
                    size_t t2 = ln.find('\t', t1 + 1);
                    region_genome += atoll(ln.c_str() + t2 + 1) - atoll(ln.c_str() + t1 + 1);
                }
            }
            genome = region_genome;
        }
        const double coverage = (1 - pBad) * (double)J.mapped * rlMean / (double)genome;     // covstats.go:277
        printf("%.2f\t%.2f\t%.2f\t%d\t%d\t%.2f\t%.2f\t%.2f\t%.1f\t%.1f\t%.1f\t%d\t%s\t%s\n", coverage, insMean, insSd, pct5, pct95, tMean, tSd,
               100 * pUnmapped, 100 * pBad, 100 * pDup, 100 * pProper, maxRead, bam.c_str(), J.names.c_str());
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------ depthwed
// getNameFromFile (depthwed.go:37-46): the file's base name without a trailing .gz, then .bed, then .depth
static std::string wed_name(const std::string& path) {
    std::string nm = path.substr(path.find_last_of('/') == std::string::npos ? 0 : path.find_last_of('/') + 1);
    for (const char* suf : {".gz", ".bed", ".depth"}) if (ends_with(nm, suf)) nm = nm.substr(0, nm.size() - strlen(suf));
    return nm;
}

static void append_int(std::string& out, long long v) {
    char b[24];
    int n = 0;
    unsigned long long u = v < 0 ? 0ull - (unsigned long long)v : (unsigned long long)v;
    do { b[n++] = (char)('0' + u % 10); u /= 10; } while (u);
    if (v < 0) out.push_back('-');
    while (n) out.push_back(b[--n]);
}

// The matrix rows as depthwed.go:69-75 prints them: chrom, start, end, then every sample's cell(g, s), tab-separated.  Blocks
// of rows are formatted on the host pool, a batch of blocks at a time, and written in order.
template <class Pos, class Cell>
static void wed_write(FILE* f, int64_t G, size_t S, const std::vector<std::string>& chroms, const int32_t* oc, const Pos* os, const Pos* oe,
                      const Cell& cell) {
    const int64_t kRows = 4096;
    const int64_t nb = (G + kRows - 1) / kRows;
    glhost::ThreadPool& pool = glhost::ThreadPool::global();
    const int64_t batch = 2 * (int64_t)pool.size();
    std::vector<std::string> txt((size_t)std::min<int64_t>(batch, std::max<int64_t>(nb, 1)));
    for (int64_t b0 = 0; b0 < nb; b0 += batch) {
        const int64_t b1 = std::min(nb, b0 + batch);
        pool.run(b1 - b0, [&](int64_t t, int) {
            std::string& out = txt[(size_t)t];
            out.clear();
            const int64_t g0 = (b0 + t) * kRows, g1 = std::min(G, g0 + kRows);
            for (int64_t g = g0; g < g1; g++) {
                out += chroms[(size_t)oc[g]];
                out.push_back('\t'); append_int(out, (long long)os[g]);
                out.push_back('\t'); append_int(out, (long long)oe[g]);
                for (size_t s = 0; s < S; s++) { out.push_back('\t'); append_int(out, (long long)cell(g, s)); }
                out.push_back('\n');
            }
        });
        for (int64_t t = 0; t < b1 - b0; t++) fwrite(txt[(size_t)t].data(), 1, txt[(size_t)t].size(), f);
    }
}

// depthwed from BAMs: the matrix `goleft depth --prefix <base> -w W -Q Q [-c chrom] -r ref.fa x.bam` for every BAM, then
// `goleft depthwed -s SIZE <base>[.chrom].depth.bed ...` print, with no text in between.  The rows are the .fai windows
// [iW, min((i+1)W, len)) of every contig (or -c); the groups come from gl_depthwed_plan once, with a device map from window
// to group.  The BAMs go through a BamQueue, one worker per GPU: per contig (in passes of at most 2^30 - 1 bases) fetch,
// gl_depth_reduce, gl_depthwed_add_column into the sample's int64 column on the device; the finished column comes home once,
// as int32 cells (int64 when a group sum does not fit).  The main thread takes the BAMs' messages in argument order, and the
// first that failed ends the run before anything is printed.
namespace {

struct WedJob : BamJob {
    std::string note;                       // a line for stderr
    std::vector<int64_t> wide;              // the column as int64 when a group sum does not fit int32
    glhts::DecodeStats dec;
    int gpu_fed = 0;
    double gpu_s = 0, d2h_s = 0;
};

struct WedContig { std::string name; long long len; int64_t w0; };

}  // namespace

static int wed_bams(const ArgParser& ap, long long size, const std::string& w, const std::string& q, const std::string& reference,
                    const std::string& chrom, const std::string& procs, const std::string& gpus, bool timing) {
    const double t_start = now_s();
    const std::vector<std::string>& bams = ap.positional;
    const size_t S = bams.size();
    if (reference.empty()) ap.fail("--reference is required with BAM inputs");
    const int W = atoi(w.c_str()), Q = atoi(q.c_str()), threads = std::max(0, atoi(procs.c_str()));
    if (W <= 0) ap.fail("windowsize must be > 0");
    const long long step = std::max(1LL, 10000000LL / W) * W;                // depth.go:132
    const long long pass = pass_length(step, W, "goleft depthwed");

    // rows: the .fai contigs goleft depth walks (cmd_depth), their windows numbered across the genome
    std::vector<WedContig> contigs;
    int64_t R = 0;
    for (const std::string& ln : read_lines(reference + ".fai", true)) {
        size_t t1 = ln.find('\t');
        if (t1 == std::string::npos) continue;
        std::string c = ln.substr(0, t1);
        if (!chrom.empty() && c != chrom) continue;
        const long long len = atoll(ln.c_str() + t1 + 1);
        if (len <= 0) continue;
        contigs.push_back({c, len, R});
        R += (len + W - 1) / W;
    }
    // groups, planned contig by contig (a group never crosses a contig)
    std::vector<std::string> names;
    std::vector<int32_t> oc, grp_of((size_t)R);
    std::vector<int64_t> os, oe;
    {
        std::vector<int64_t> rs, re, first;
        std::vector<int32_t> cid;
        for (size_t c = 0; c < contigs.size(); c++) {
            const WedContig& k = contigs[c];
            const int64_t n = (k.len + W - 1) / W;
            rs.resize((size_t)n); re.resize((size_t)n); first.resize((size_t)n + 1); cid.assign((size_t)n, (int32_t)c);
            for (int64_t i = 0; i < n; i++) { rs[(size_t)i] = i * W; re[(size_t)i] = std::min<int64_t>((i + 1) * W, k.len); }
            const size_t g0 = os.size();
            os.resize(g0 + (size_t)n); oe.resize(os.size()); oc.resize(os.size());
            int64_t ng = 0;
            if (gl_depthwed_plan(rs.data(), re.data(), cid.data(), n, size, first.data(), os.data() + g0, oe.data() + g0, oc.data() + g0, n, &ng) != GL_OK)
                fatal(1, "gl_depthwed_plan: %s", gl_last_error(nullptr));
            os.resize(g0 + (size_t)ng); oe.resize(os.size()); oc.resize(os.size());
            if (os.size() > (size_t)INT32_MAX) fatal(1, "goleft depthwed: more than 2^31 - 1 output rows");
            for (int64_t g = 0; g < ng; g++)
                std::fill(grp_of.begin() + (k.w0 + first[(size_t)g]), grp_of.begin() + (k.w0 + first[(size_t)g + 1]), (int32_t)(g0 + (size_t)g));
            names.push_back(k.name);
        }
    }
    const int64_t G = (int64_t)os.size();
    std::string header = "#chrom\tstart\tend";
    const std::string sfx = chrom.empty() ? "" : "." + chrom;                 // depth.go:378-389
    for (const std::string& b : bams) {
        std::string base = b.substr(b.find_last_of('/') == std::string::npos ? 0 : b.find_last_of('/') + 1);
        base = base.substr(0, base.size() - 4);                               // every input ends in .bam
        header += "\t" + wed_name(base + sfx + ".depth.bed");
    }
    if (G == 0) {                                   // no windows (-c names no .fai contig): the header alone, once every BAM opens
        for (const std::string& b : bams) {
            glhts::BamFile f;
            const std::string e = f.open(b);
            if (!e.empty()) fatal(1, "%s", e.c_str());
        }
        printf("%s\n", header.c_str());
        return 0;
    }

    const GpuPlan gp = resolve_gpus(gpus, S, "goleft depthwed");
    std::vector<int32_t> m32((size_t)S * (size_t)G);                          // sample-major: column s at [s * G, (s + 1) * G)
    BamQueue<WedJob> queue(bams);
    struct Dev { gl_ctx* c = nullptr; int32_t* map = nullptr; int64_t* col = nullptr; int32_t* col32 = nullptr; int32_t* ovf = nullptr; };
    // BAM i on one worker's device: its column into m32 (or J.wide)
    auto run = [&](Dev& d, size_t i, gl_bam*) {
        WedJob& J = queue.jobs[i];
        gl_ctx* c = d.c;
        gl_bam& bam = *J.bh;
        glhts::SegmentSet whole;
        SegSource src;
        std::map<std::string, int> tid_of;
        for (size_t r = 0; r < bam.f.header.refs.size(); r++) tid_of[bam.f.header.refs[r].name] = (int)r;
        int only = -1;
        if (!chrom.empty()) { auto it = tid_of.find(chrom); if (it != tid_of.end()) only = it->second; }
        const int thr = threads > 0 ? threads : (int)std::max(1u, std::thread::hardware_concurrency());
        const double t0 = now_s();
        std::string e;
        if (decode_unindexed(bam.f, bams[i], Q, thr, only, whole, e)) {
            J.note = "goleft depthwed: no usable index (.bai or .csi) next to " + bams[i] + ": decoding the whole file";
            if (!e.empty()) { J.code = 1; J.msg = e; return; }
            src.whole = &whole;
            J.dec.wall_s += now_s() - t0;
        }
        glck(c, gl_depthwed_column_begin(c, d.col, G), "gl_depthwed_column_begin");
        for (const WedContig& k : contigs) {
            auto it = tid_of.find(k.name);
            if (it == tid_of.end()) continue;                                 // not in the BAM: every window is 0
            for (long long ps = 0; ps < k.len; ps += pass) {
                const long long pe = std::min(k.len, ps + pass);
                src.fetch_pass(c, bam, it->second, ps, pe, k.len, Q, threads, &J.dec, &J.gpu_fed);
                const double tg = now_s();
                glck(c, gl_depth_begin(c, ps, pe), "gl_depth_begin");
                src.add(c);
                glck(c, gl_depth_reduce(c, W, 4, 0, step), "gl_depth_reduce");
                glck(c, gl_depthwed_add_column(c, k.w0 + ps / W, d.map, d.col), "gl_depthwed_add_column");
                J.gpu_s += now_s() - tg;
            }
        }
        const double t1 = now_s();
        glck(c, gl_depthwed_column_i32(c, d.col, G, d.col32, d.ovf), "gl_depthwed_column_i32");
        int32_t ovf = 0;
        if (G) glck(c, gl_memcpy_d2h(c, m32.data() + i * (size_t)G, d.col32, G * 4), "gl_memcpy_d2h");
        glck(c, gl_memcpy_d2h(c, &ovf, d.ovf, 4), "gl_memcpy_d2h");
        if (ovf) {
            J.wide.resize((size_t)G);
            glck(c, gl_memcpy_d2h(c, J.wide.data(), d.col, G * 8), "gl_memcpy_d2h");
        }
        J.d2h_s = now_s() - t1;
    };
    queue.start(gp, [&](int g, std::string& err) {
        Dev d;
        if (gl_ctx_create(g % gp.n_dev, &d.c) != GL_OK) { err = std::string("goleft depthwed: gl_ctx_create: ") + gl_last_error(nullptr); return d; }
        void *pm = nullptr, *pc = nullptr, *p32 = nullptr, *po = nullptr;
        if (gl_dev_alloc(d.c, std::max<int64_t>(R, 1) * 4, &pm) != GL_OK || gl_dev_alloc(d.c, std::max<int64_t>(G, 1) * 8, &pc) != GL_OK ||
            gl_dev_alloc(d.c, std::max<int64_t>(G, 1) * 4, &p32) != GL_OK || gl_dev_alloc(d.c, 16, &po) != GL_OK ||
            (R > 0 && gl_memcpy_h2d(d.c, pm, grp_of.data(), R * 4) != GL_OK))
            err = std::string("goleft depthwed: goleft depthwed: ") + gl_last_error(d.c);
        d.map = static_cast<int32_t*>(pm); d.col = static_cast<int64_t*>(pc); d.col32 = static_cast<int32_t*>(p32); d.ovf = static_cast<int32_t*>(po);
        return d;
    }, run, [](Dev& d) {
        for (void* p : std::initializer_list<void*>{d.map, d.col, d.col32, d.ovf}) if (p) gl_dev_free(d.c, p);
        gl_ctx_destroy(d.c);
    });
    for (size_t i = 0; i < S; i++) {
        const WedJob& J = queue.wait(i);
        if (!J.note.empty()) fprintf(stderr, "%s\n", J.note.c_str());
        if (J.code) { queue.stop(); fatal(J.code, "%s", J.msg.c_str()); }
    }
    queue.stop();
    const double t_fmt = now_s();
    printf("%s\n", header.c_str());
    wed_write(stdout, G, S, names, oc.data(), os.data(), oe.data(), [&](int64_t g, size_t s) -> long long {
        const WedJob& J = queue.jobs[s];
        return J.wide.empty() ? (long long)m32[s * (size_t)G + (size_t)g] : (long long)J.wide[(size_t)g];
    });
    fflush(stdout);
    if (timing) {
        double dec = 0, gpu = 0, d2h = 0; long long rec = 0, bin = 0; int fed = 0;
        for (const WedJob& J : queue.jobs) { dec += J.dec.wall_s; gpu += J.gpu_s; d2h += J.d2h_s; rec += J.dec.n_records; bin += J.dec.bytes_in; fed += J.gpu_fed; }
        fprintf(stderr, "{\"goleft_depthwed_timing\": {\"wall_s\": %.4f, \"gpus\": %d, \"samples\": %zu, \"windows\": %lld, \"rows\": %lld, "
                        "\"decode_wall_s_sum\": %.4f, \"reduce_column_s_sum\": %.4f, \"d2h_s_sum\": %.4f, \"format_s\": %.4f, "
                        "\"records\": %lld, \"bgzf_bytes_in\": %lld, \"gpu_fed_passes\": %d}}\n",
                now_s() - t_start, gp.G, S, (long long)R, (long long)G, dec, gpu, d2h, now_s() - t_fmt, rec, bin, fed);
    }
    return 0;
}

static int cmd_depthwed(int argc, char** argv) {
    std::string size, w = "250", q = "1", reference, chrom, procs = "0", gpus = "0", bed;
    bool timing = false;
    ArgParser ap;
    ap.prog = "goleft depthwed";
    ap.add("size", 's', &size, true);
    // extension: BAM inputs, with goleft depth's options and defaults
    ap.add("windowsize", 'w', &w); ap.add("q", 'Q', &q); ap.add("reference", 'r', &reference); ap.add("chrom", 'c', &chrom);
    ap.add("processes", 'p', &procs); ap.add("gpus", 0, &gpus); ap.addb("timing", 0, &timing);
    ap.add("bed", 'b', &bed);
    ap.parse(argc, argv);
    if (ap.positional.empty()) ap.fail("beds is required");
    const long long sz = atoll(size.c_str());
    size_t n_bam = 0;
    for (const std::string& p : ap.positional) n_bam += ends_with(p, ".bam");
    if (n_bam && n_bam < ap.positional.size()) ap.fail("inputs must be all BAMs or all depth.bed files");
    if (ap.given("bed")) ap.fail("--bed is not supported: BAM inputs are windowed over the .fai contigs of --reference");
    if (n_bam) return wed_bams(ap, sz, w, q, reference, chrom, procs, gpus, timing);
    for (const char* f : {"windowsize", "q", "reference", "chrom", "processes", "gpus", "timing"})
        if (ap.given(f)) ap.fail(std::string("--") + f + " needs BAM inputs");
    const size_t S = ap.positional.size();
    std::vector<std::string> chroms;
    std::map<std::string, int> chrom_id;
    std::vector<int32_t> starts, ends, cid;
    std::vector<double> means;                       // kept only for the rare case a depth does not fit int32
    std::vector<int32_t> depth32;                    // int(0.5 + mean), rounded where the reference rounds: at parse time (depthwed.go:103)
    bool fits32 = true;
    size_t R = 0;
    std::string header = "#chrom\tstart\tend";
    for (size_t f = 0; f < S; f++) {
        header += "\t" + wed_name(ap.positional[f]);
        std::vector<std::string> lines = read_lines(ap.positional[f], true);
        if (f == 0) { R = lines.size(); means.resize(S * R); depth32.resize(S * R); }
        else if (lines.size() != R) fatal(2, "panic: not all files have same number of records");
        for (size_t r = 0; r < R; r++) {
            const std::string& ln = lines[r];
            size_t t1 = ln.find('\t'), t2 = ln.find('\t', t1 + 1), t3 = ln.find('\t', t2 + 1);
            if (t1 == std::string::npos || t2 == std::string::npos || t3 == std::string::npos) fatal(1, "bad line in %s: %s", ap.positional[f].c_str(), ln.c_str());
            const double dep = strtod(ln.c_str() + t3 + 1, nullptr);
            means[f * R + r] = dep;
            const double rd = 0.5 + dep;                                            // Go: int(0.5 + dep) truncates toward zero
            if (!(rd > -2147483648.0 && rd < 2147483648.0)) fits32 = false;
            else depth32[f * R + r] = (int32_t)rd;
            if (f == 0) {
                std::string c = ln.substr(0, t1);
                auto it = chrom_id.find(c);
                if (it == chrom_id.end()) { it = chrom_id.emplace(c, (int)chroms.size()).first; chroms.push_back(c); }
                cid.push_back(it->second);
                starts.push_back(atoi(ln.c_str() + t1 + 1));
                ends.push_back(atoi(ln.c_str() + t2 + 1));
            }
        }
    }
    printf("%s\n", header.c_str());
    if (R == 0) return 0;
    gl_ctx* ctx = open_ctx(0, "goleft depthwed");
    std::vector<int32_t> os(R), oe(R), oc(R);
    std::vector<int64_t> out;
    std::vector<int32_t> out32;
    int64_t n_out = 0;
    bool have32 = false;
    if (fits32) {                                    // 4 B in + 4 B out per cell; a group sum beyond int32 falls through to the 64-bit path
        out32.resize(R * S);
        const int rc = gl_depthwed_aggregate_i32(ctx, depth32.data(), (int32_t)S, (int64_t)R, starts.data(), ends.data(), cid.data(), sz, os.data(),
                                                 oe.data(), oc.data(), out32.data(), (int64_t)R, &n_out);
        if (rc == GL_OK) have32 = true;
        else if (!(rc == GL_ERANGE && n_out == -1)) glck(ctx, rc, "gl_depthwed_aggregate_i32");
    }
    if (!have32) {
        out.resize(R * S);
        glck(ctx, gl_depthwed_aggregate(ctx, means.data(), (int32_t)S, (int64_t)R, starts.data(), ends.data(), cid.data(), sz, os.data(), oe.data(),
                                        oc.data(), out.data(), (int64_t)R, &n_out), "gl_depthwed_aggregate");
    }
    wed_write(stdout, n_out, S, chroms, oc.data(), os.data(), oe.data(), [&](int64_t g, size_t s) -> long long {
        return have32 ? (long long)out32[(size_t)g * S + s] : (long long)out[(size_t)g * S + s];
    });
    gl_ctx_destroy(ctx);
    return 0;
}

// ------------------------------------------------------------------------------------------------ indexsplit
// indexsplit/indexsplit.go:24-30,197-216: N regions of about equal amounts of data across the cohort, from the indexes alone
static int cmd_indexsplit(int argc, char** argv) {
    std::string n, fai, problematic;
    ArgParser ap;
    ap.prog = "goleft indexsplit";
    ap.add("n", 'n', &n, true); ap.add("fai", 0, &fai); ap.add("problematic", 'p', &problematic);
    ap.parse(argc, argv);
    if (ap.positional.empty()) ap.fail("indexes is required");
    const std::vector<std::string>& paths = ap.positional;
    const int N = atoi(n.c_str());

    // references: from the first BAM's header, else from the .fai (the reference's ReadFai references carry ID -1 and
    // Split indexes a slice with it; here a .fai reference's id is its position in the file)
    struct Ref { std::string name; int64_t len; int id; };
    std::vector<Ref> refs;
    if (ends_with(paths[0], ".bam")) {
        glhts::BamHeader h;
        std::string e = glhts::bam_read_header(paths[0], h);
        if (!e.empty()) fatal(1, "%s", e.c_str());
        for (size_t i = 0; i < h.refs.size(); i++) refs.push_back({h.refs[i].name, h.refs[i].length, (int)i});
    } else {
        std::vector<glhts::RefInfo> r;
        std::string e = glhts::fai_read(fai, r);
        if (!e.empty()) fatal(1, "error opening fai: %s. Is is present?", fai.c_str());
        std::stable_sort(r.begin(), r.end(), [](const glhts::RefInfo& a, const glhts::RefInfo& b) { return a.offset < b.offset; });   // indexcov.go:293
        for (auto& x : r) refs.push_back({x.name, x.length, (int)refs.size()});
    }
    const int32_t R = (int32_t)refs.size();

    gl_ctx* ctx = open_ctx(0, "goleft indexsplit");
    const size_t S = paths.size();
    std::vector<int64_t> all_sizes, ptr(S * (size_t)(R + 1), 0), max_len((size_t)R, 0);
    for (size_t i = 0; i < S; i++) {                                        // indexcov.ReadIndex(path).Sizes(), indexsplit.go:92-93
        const std::string& b = paths[i];
        std::vector<int64_t> sz, sp;
        if (ends_with(b, ".crai")) {
            std::vector<glhts::CraiSlices> cr;
            std::string e = glhts::crai_read(b, cr);
            if (!e.empty()) fatal(1, "%s", e.c_str());
            crai_sizes(cr, sz, sp);
        } else {
            glhts::BaiIndex bai;
            std::string e = glhts::bai_read(bai_path(b), bai);
            if (!e.empty()) fatal(1, "%s", e.c_str());
            refuse_wide_csi(bai, bai_path(b), "indexsplit");
            const size_t nr = bai.ioffsets.size();
            std::vector<uint64_t> voff;
            std::vector<int64_t> rp(nr + 1, 0);
            for (size_t r = 0; r < nr; r++) { voff.insert(voff.end(), bai.ioffsets[r].begin(), bai.ioffsets[r].end()); rp[r + 1] = (int64_t)voff.size(); }
            sz.resize(voff.size() + 1); sp.assign(nr + 1, 0);
            glck(ctx, gl_indexcov_sizes(ctx, voff.data(), rp.data(), (int32_t)nr, sz.data(), sp.data()), "gl_indexcov_sizes");
            sz.resize((size_t)sp[nr]);
        }
        if (sp.back() < 1) fatal(1, "indexcov: no usable chromsomes in bam: %s", b.c_str());     // Index.init, indexcov.go:100-102
        const int64_t base = (int64_t)all_sizes.size();
        const int32_t nr = (int32_t)sp.size() - 1;
        for (int32_t r = 0; r <= R; r++) ptr[i * (size_t)(R + 1) + r] = base + sp[(size_t)std::min(r, nr)];
        for (int32_t r = 0; r < R && r < nr; r++) max_len[(size_t)r] = std::max(max_len[(size_t)r], sp[(size_t)r + 1] - sp[(size_t)r]);
        all_sizes.insert(all_sizes.end(), sz.begin(), sz.begin() + sp[(size_t)std::min(R, nr)]);
    }
    std::vector<int64_t> out_ptr((size_t)R + 1, 0);
    for (int32_t r = 0; r < R; r++) out_ptr[(size_t)r + 1] = out_ptr[(size_t)r] + max_len[(size_t)r];
    std::vector<double> tile_sum((size_t)out_ptr[(size_t)R] + 1, 0.0);
    glck(ctx, gl_indexsplit_accumulate(ctx, all_sizes.data(), ptr.data(), (int32_t)S, R, out_ptr.data(), tile_sum.data()), "gl_indexsplit_accumulate");

    // -p: BED of problematic regions (depth.ReadTree, depth/intervals.go:42-82)
    std::vector<int32_t> pr; std::vector<int64_t> ps, pe;
    if (!problematic.empty()) {
        std::map<std::string, int> num;
        for (int32_t q = 0; q < R; q++) num.emplace(refs[(size_t)q].name, q);
        for (const std::string& ln : read_lines(problematic, true)) {
            std::string c; long long s0, e0;
            if (!chrom_start_end(ln, c, s0, e0)) fatal(2, "panic: couldn't get region from line %s", ln.c_str());
            if (s0 >= e0) continue;
            auto it = num.find(c);
            if (it != num.end()) { pr.push_back(it->second); ps.push_back(s0); pe.push_back(e0); }
        }
    }
    std::vector<const char*> nm; std::vector<int64_t> ln_; std::vector<int32_t> ids;
    for (const Ref& r : refs) { nm.push_back(r.name.c_str()); ln_.push_back(r.len); ids.push_back(r.id); }
    char* text = nullptr; int64_t tl = 0;
    if (gl_indexsplit_chunks(tile_sum.data(), out_ptr.data(), R, nm.data(), ln_.data(), ids.data(), R, N, pr.data(), ps.data(), pe.data(),
                             (int64_t)pr.size(), &text, &tl) != GL_OK) fatal(1, "gl_indexsplit_chunks failed");
    fwrite(text, 1, (size_t)tl, stdout);
    gl_free_text(text);
    gl_ctx_destroy(ctx);
    return 0;
}

// ------------------------------------------------------------------------------------------------ multidepth
// multidepth/multidepth.go: blocks of one chromosome where more than --minsamples of the BAMs reach --mincov, with every
// sample's mean depth.  Two passes over each sample's segments on the GPU (counts, then block sums); the segments are
// decoded once and kept in their compact form in between (packed8 words, or the GPU feeder's int32 copied to pinned memory).
// With --gpus, each worker (one gl_ctx per GPU) counts its own range of samples; worker 0 merges the others' per-base
// counters (gl_multidepth_merge) and finds the sites, and every worker sums its samples against the same blocks.
// The output is the reference's with -p 1 (chunks in order), whatever the number of workers.
static int cmd_multidepth(int argc, char** argv) {
    std::string q = "10", chrom, mincov = "7", maxcov = "1000", maxskip = "10", minsize = "15", window = "10000000", procs = "0",
                minsamples = "0.5", gpus = "0";
    ArgParser ap;
    ap.prog = "goleft multidepth";
    ap.add("q", 'Q', &q); ap.add("chrom", 'c', &chrom, true); ap.add("mincov", 0, &mincov); ap.add("maxcov", 0, &maxcov);
    ap.add("maxskip", 'k', &maxskip); ap.add("minsize", 'm', &minsize); ap.add("window", 'w', &window); ap.add("processes", 'p', &procs);
    ap.add("minsamples", 0, &minsamples);
    ap.add("gpus", 0, &gpus);                       // extension: GPUs to use (0 = every visible one); samples are sharded over them
    ap.parse(argc, argv);
    if (ap.positional.empty()) ap.fail("bams is required");
    const std::vector<std::string>& bams = ap.positional;
    const int S = (int)bams.size();
    const int Q = atoi(q.c_str()), threads = std::max(0, atoi(procs.c_str()));     // --maxcov: accepted, no effect (DESIGN §0)
    // header: the short name of every BAM (multidepth.go:66-72); the contig length from the first (chromSize, :34-48)
    std::string hdr = "#chrom\tstart\tend";
    std::vector<gl_bam> bam((size_t)S);
    std::vector<int> tid((size_t)S, -1);
    long long L = -1;
    for (int i = 0; i < S; i++) {
        std::string e = bam[(size_t)i].f.open(bams[(size_t)i]);
        if (!e.empty()) fatal(2, "panic: %s", e.c_str());
        hdr += "\t" + short_name(bams[(size_t)i], false, &bam[(size_t)i].f.header);
        const auto& refs = bam[(size_t)i].f.header.refs;
        for (size_t r = 0; r < refs.size(); r++) if (refs[r].name == chrom) { tid[(size_t)i] = (int)r; if (i == 0) L = refs[r].length; }
        if (tid[(size_t)i] < 0) fatal(2, "panic: multidepth: chromosome %s not found in %s", chrom.c_str(), bams[(size_t)i].c_str());
    }
    // --gpus: the samples in contiguous ranges, one per worker, balanced by each sample's compressed bytes of the contig (the
    // linear-index offsets of its first and last tile), or by file size without an index.  Any split prints the same bytes.
    const GpuPlan gp = resolve_gpus(gpus, (size_t)S, "goleft multidepth");
    if (L <= 0) { printf("%s\n", hdr.c_str()); return 0; }
    std::vector<int> lo((size_t)gp.G + 1, S);
    {
        std::vector<double> pre((size_t)S + 1, 0.0);
        for (int i = 0; i < S; i++) {
            const glhts::BamFile& f = bam[(size_t)i].f;
            double w = -1;
            if (f.has_index && tid[(size_t)i] < (int)f.bai.ioffsets.size()) {
                uint64_t a = 0, b = 0;
                for (uint64_t v : f.bai.ioffsets[(size_t)tid[(size_t)i]]) if (v) { if (!a) a = v; b = v; }
                if (a) w = (double)((b >> 16) - (a >> 16) + 1);
            }
            if (w < 0) { struct stat sb; w = stat(bams[(size_t)i].c_str(), &sb) == 0 ? (double)sb.st_size : 1.0; }
            pre[(size_t)i + 1] = pre[(size_t)i] + std::max(w, 1.0);
        }
        lo[0] = 0;
        for (int g = 1; g < gp.G; g++) {
            const double target = pre[(size_t)S] * g / gp.G;
            int i = lo[(size_t)g - 1] + 1;
            while (i < S - (gp.G - g) && pre[(size_t)i] < target) i++;
            lo[(size_t)g] = i;
        }
    }
    const int mc = atoi(mincov.c_str());
    const double ms = atof(minsamples.c_str());
    std::vector<SegSource> smp((size_t)S);
    std::vector<glhts::SegmentSet> whole((size_t)S);
    std::vector<gl_ctx*> ctx((size_t)gp.G, nullptr);
    std::vector<std::vector<void*>> pinned((size_t)gp.G);
    // sample i's segments of the contig: without an index, a whole-file decode of that one reference; otherwise the GPU feeder
    // when it can, else the host feeder.  A sample that stays on the host is decoded on a helper thread beside the GPU work
    // of sample i-1.
    auto stays_on_host = [&](int i) { return !(SegSource::gpu_feed() && index_usable(bam[(size_t)i].f)); };
    auto fetch = [&](gl_ctx* c, int i) {
        const size_t k = (size_t)i;
        std::string e;
        if (decode_unindexed(bam[k].f, bams[k], Q, threads > 0 ? threads : 8, tid[k], whole[k], e)) {
            if (!e.empty()) fatal(1, "%s", e.c_str());
            smp[k].whole = &whole[k];
        }
        smp[k].fetch(c, bam[k], tid[k], 0, L, Q, threads, 0, true, nullptr, nullptr);
    };
    // pass 1, per worker over its samples
    for (std::thread& t : start_workers(gp, [&](int g) {
             gl_ctx* c = ctx[(size_t)g] = open_ctx(g % gp.n_dev, "goleft multidepth");
             glck(c, gl_multidepth_begin(c, L, S, mc, ms), "goleft multidepth");
             const int i0 = lo[(size_t)g], i1 = lo[(size_t)g + 1];
             std::thread next;
             bool next_host = false;
             for (int i = i0; i < i1; i++) {
                 SegSource& m = smp[(size_t)i];
                 if (next.joinable()) next.join();
                 if (!next_host) fetch(c, i);
                 next_host = i + 1 < i1 && stays_on_host(i + 1);
                 if (next_host) next = std::thread(fetch, c, i + 1);
                 glck(c, gl_depth_begin(c, 0, L), "gl_depth_begin");
                 m.add(c);
                 glck(c, gl_multidepth_count(c), "gl_multidepth_count");
                 if (m.on_device) {                  // pass 2 needs the feeder's arrays after the next decode reuses them
                     void* p = nullptr;
                     glck(c, gl_host_alloc_pinned(c, std::max<int64_t>(m.n, 1) * 8, &p), "gl_host_alloc_pinned");
                     pinned[(size_t)g].push_back(p);
                     int32_t* pin = static_cast<int32_t*>(p);
                     if (m.n > 0) {
                         glck(c, gl_memcpy_d2h(c, pin, m.s, m.n * 4), "gl_memcpy_d2h");
                         glck(c, gl_memcpy_d2h(c, pin + m.n, m.e, m.n * 4), "gl_memcpy_d2h");
                     }
                     m.view(pin, pin + m.n, m.n);
                 }
             }
             if (next.joinable()) next.join();
         }))
        t.join();
    // worker 0 adds up every worker's counts, then the blocks
    if (gp.G > 1) glck(ctx[0], gl_multidepth_merge(ctx[0], ctx.data() + 1, gp.G - 1), "gl_multidepth_merge");
    int64_t nr = 0;
    glck(ctx[0], gl_multidepth_sites(ctx[0], nullptr, nullptr, 0, &nr), "gl_multidepth_sites");
    std::vector<int32_t> rs((size_t)std::max<int64_t>(nr, 1));
    std::vector<uint8_t> rc((size_t)std::max<int64_t>(nr, 1));
    glck(ctx[0], gl_multidepth_sites(ctx[0], rs.data(), rc.data(), nr, &nr), "gl_multidepth_sites");
    const int64_t max_skip = atoll(maxskip.c_str()), min_size = atoll(minsize.c_str()), win = atoll(window.c_str());
    int64_t nb = 0;
    if (gl_multidepth_blocks(rs.data(), rc.data(), nr, L, S, 0, max_skip, min_size, win, nullptr, nullptr, nullptr, 0, &nb) != GL_OK)
        fatal(1, "gl_multidepth_blocks failed");
    std::vector<int64_t> bs((size_t)std::max<int64_t>(nb, 1)), be(bs.size()), bn(bs.size());
    if (gl_multidepth_blocks(rs.data(), rc.data(), nr, L, S, 0, max_skip, min_size, win, bs.data(), be.data(), bn.data(), nb, &nb) != GL_OK)
        fatal(1, "gl_multidepth_blocks failed");
    // pass 2: every other worker takes worker 0's sites; the samples keep their cohort numbers
    for (std::thread& t : start_workers(gp, [&](int g) {
             gl_ctx* c = ctx[(size_t)g];
             if (g > 0) glck(c, gl_multidepth_adopt_sites(c, ctx[0]), "gl_multidepth_adopt_sites");
             glck(c, gl_multidepth_set_blocks(c, bs.data(), be.data(), bn.data(), nb), "gl_multidepth_set_blocks");
             for (int i = lo[(size_t)g]; i < lo[(size_t)g + 1]; i++) {
                 glck(c, gl_depth_begin(c, 0, L), "gl_depth_begin");
                 smp[(size_t)i].add(c);
                 glck(c, gl_multidepth_sums(c, i), "gl_multidepth_sums");
             }
         }))
        t.join();
    const size_t cells = (size_t)nb * (size_t)S;
    std::vector<int64_t> qv(std::max<size_t>(cells, 1));
    std::vector<double> val(qv.size());
    std::vector<uint8_t> cert(qv.size());
    glck(ctx[0], gl_multidepth_result(ctx[0], nullptr, qv.data(), val.data(), cert.data()), "gl_multidepth_result");
    if (gp.G > 1) {                                 // each sample's columns from the worker that summed it
        std::vector<int64_t> tq(qv.size());
        std::vector<double> tv(qv.size());
        std::vector<uint8_t> tc(qv.size());
        for (int g = 1; g < gp.G; g++) {
            glck(ctx[(size_t)g], gl_multidepth_result(ctx[(size_t)g], nullptr, tq.data(), tv.data(), tc.data()), "gl_multidepth_result");
            for (size_t r = 0; r < (size_t)nb; r++)
                for (size_t k = r * S + lo[(size_t)g]; k < r * S + lo[(size_t)g + 1]; k++) { qv[k] = tq[k]; val[k] = tv[k]; cert[k] = tc[k]; }
        }
    }
    char* text = nullptr;
    int64_t tl = 0;
    if (gl_multidepth_text(chrom.c_str(), bs.data(), be.data(), nb, S, qv.data(), val.data(), cert.data(), threads, &text, &tl) != GL_OK)
        fatal(1, "gl_multidepth_text failed");
    printf("%s\n", hdr.c_str());
    fwrite(text, 1, (size_t)tl, stdout);
    gl_free_text(text);
    for (int g = 0; g < gp.G; g++) {
        for (void* p : pinned[(size_t)g]) gl_host_free_pinned(ctx[(size_t)g], p);
        gl_ctx_destroy(ctx[(size_t)g]);
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------ samplename
// samplename/samplename.go: one @RG -> its SM (nothing when empty); several -> the distinct non-empty SMs, here in header
// order (the reference iterates a Go map).  -e: anything but exactly one sample is an error.
static int cmd_samplename(int argc, char** argv) {
    bool err_multi = false;
    ArgParser ap;
    ap.prog = "goleft samplename";
    ap.addb("errormulti", 'e', &err_multi);
    ap.parse(argc, argv);
    if (ap.positional.empty()) ap.fail("bam is required");
    glhts::BamHeader h;
    std::string e = glhts::bam_read_header(ap.positional[0], h);
    if (!e.empty()) fatal(2, "panic: %s", e.c_str());
    const std::vector<std::string> names = h.sample_names();
    if (err_multi && names.size() != 1) fatal(2, "panic: goleft/samplename: found multiple samples in %s", ap.positional[0].c_str());
    std::string out;
    for (size_t i = 0; i < names.size(); i++) out += (i ? "\n" : "") + names[i];
    printf("%s\n", out.c_str());
    return 0;
}

// ------------------------------------------------------------------------------------------------ dcnv
// dcnv/dcnv.go:153-186,323-354 (a separate binary of the reference; `dcnv <matrix> <ref.fa>`, positional only): read the
// sites x samples matrix depthwed writes (plain, gzip/BGZF or "-"), take each row's GC from the FASTA, argsort the rows by
// GC as Go does (gl_go_argsort_f64), debias and median-normalise every sample on the GPU (gl_dcnv_normalize, column blocks
// sized to device memory), and write depth.bed with "%.2f" tokens made on the GPU (gl_format_f2).  The reference's panics
// are an error message and exit 2.  Parsing and row assembly run on the host pool.
// `dcnv --svd PCT` (also --svd=PCT, before the positionals; DESIGN §1.13) then removes the cohort's leading components from
// the normalised matrix (gl_dcnv_svd, row blocks sized to device memory) and logs "variance:" with the removed ones' shares.
// PCT must be finite and >= 0, else exit 255 as go-arg's flag errors.
// `dcnv --chunk W` (also --chunk=W; DESIGN §1.9) debiases with the reference's unreached ChunkDebiaser in place of the
// moving median: the GC-sorted rows are cut into chunks spanning at most W of GC (gl_dcnv_chunk_slices), and each sample's
// values in a chunk are divided by their median there (gl_dcnv_normalize_chunked).  W must be finite and > 0, else exit 255.
namespace {

struct DcnvRow { const char* p; size_t n; };                 // one line, without its "\n"

bool go_space(char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '\v' || c == '\f'; }

// strconv.Atoi, then the reference's uint32(); a value outside uint32 (which the reference wraps) is an error here
bool dcnv_atou32(const char* p, size_t n, int64_t& v) {
    size_t i = (n && (p[0] == '+' || p[0] == '-')) ? 1 : 0;
    if (i == n || n - i > 18) return false;
    int64_t x = 0;
    for (size_t k = i; k < n; k++) {
        if (p[k] < '0' || p[k] > '9') return false;
        x = x * 10 + (p[k] - '0');
    }
    v = p[0] == '-' ? -x : x;
    return v >= 0 && v < (int64_t(1) << 32);
}

// strconv.ParseFloat of the decimal form (depthwed writes integers: those take the fast path); NaN, Inf, hexadecimal
// and out-of-range tokens are errors here
bool dcnv_atof(const char* p, size_t n, double& v) {
    size_t i = (n && (p[0] == '+' || p[0] == '-')) ? 1 : 0;
    size_t k = i;
    while (k < n && p[k] >= '0' && p[k] <= '9') k++;
    if (k == n && k > i && k - i <= 15) {                       // at most 15 digits: exact in float64
        int64_t x = 0;
        for (size_t j = i; j < n; j++) x = x * 10 + (p[j] - '0');
        v = p[0] == '-' ? -(double)x : (double)x;
        return true;
    }
    const size_t int_digits = k - i;
    size_t frac_digits = 0;
    if (k < n && p[k] == '.') { k++; while (k < n && p[k] >= '0' && p[k] <= '9') { k++; frac_digits++; } }
    if (int_digits + frac_digits == 0) return false;
    if (k < n && (p[k] == 'e' || p[k] == 'E')) {
        k++;
        if (k < n && (p[k] == '+' || p[k] == '-')) k++;
        const size_t e0 = k;
        while (k < n && p[k] >= '0' && p[k] <= '9') k++;
        if (k == e0) return false;
    }
    if (k != n) return false;
    std::string s(p, n);
    v = strtod(s.c_str(), nullptr);                             // correctly rounded, as ParseFloat
    return std::isfinite(v);
}

// Go's log.Println prefix: "2009/11/10 23:00:00 "
void go_log(const char* msg) {
    time_t t = time(nullptr);
    struct tm tm;
    localtime_r(&t, &tm);
    fprintf(stderr, "%04d/%02d/%02d %02d:%02d:%02d %s\n", tm.tm_year + 1900, tm.tm_mon + 1, tm.tm_mday, tm.tm_hour, tm.tm_min, tm.tm_sec, msg);
}


// The sites x samples matrix depthwed writes, read by dcnv and emdepth (dcnv.go:59-104 ReadRegions): plain, gzip/BGZF or "-".
// ReadString('\n'): a final line without "\n" is dropped.  Header lines ('#' or "chrom") count only before the first data
// line, and the last one names the samples.  Every reference panic is exit 2.
struct Matrix {
    std::string text;
    std::vector<DcnvRow> rows;                               // data lines, without their "\n"
    std::vector<std::string> header;                         // the header line's fields (trimmed)
    std::vector<std::string> samples;                        // header[3:]
    std::vector<double> X;                                   // matrix_parse: rows x samples, row-major
    std::vector<int64_t> starts, ends;                       // as parsed (uint32 range)
    std::vector<std::pair<const char*, size_t>> chrom;       // into text
};

// the whole of a plain, gzip/BGZF or "-" (stdin) file, as xopen.Ropen reads it; a failure is the reference's panic (exit 2)
std::string read_whole(const std::string& path) {
    std::string text;
    gzFile f = path == "-" ? gzdopen(dup(0), "rb") : gzopen(path.c_str(), "rb");
    if (!f) fatal(2, "panic: open %s: %s", path.c_str(), strerror(errno));
    gzbuffer(f, 1 << 20);
    std::vector<char> buf((size_t)1 << 22);
    int n;
    while ((n = gzread(f, buf.data(), (unsigned)buf.size())) > 0) text.append(buf.data(), (size_t)n);
    if (n < 0) fatal(2, "panic: read %s", path.c_str());
    gzclose(f);
    return text;
}

void matrix_read(const std::string& path, Matrix& m) {
    m.text = read_whole(path);
    const std::string& text = m.text;
    bool have_header = false;
    for (size_t a = 0; a < text.size();) {
        const char* nl = static_cast<const char*>(memchr(text.data() + a, '\n', text.size() - a));
        if (!nl) break;
        const size_t b = (size_t)(nl - text.data());
        if (m.rows.empty() && (text[a] == '#' || text.compare(a, 5, "chrom") == 0)) {       // only before the first data line
            size_t s = a, e = b + 1;
            while (s < e && go_space(text[s])) s++;
            while (e > s && go_space(text[e - 1])) e--;
            std::vector<std::string> f;
            for (size_t x = s;;) {
                const size_t t = text.find('\t', x);
                if (t == std::string::npos || t >= e) { f.push_back(text.substr(x, e - x)); break; }
                f.push_back(text.substr(x, t - x));
                x = t + 1;
            }
            if (f.size() < 3) fatal(2, "panic: runtime error: slice bounds out of range (header line has %zu fields)", f.size());
            m.samples.assign(f.begin() + 3, f.end());
            m.header = std::move(f);
            have_header = true;
        } else {
            m.rows.push_back({text.data() + a, b - a});
        }
        a = b + 1;
    }
    if (!have_header) fatal(2, "panic: runtime error: integer divide by zero (no header line: no samples)");
    if (m.samples.empty()) fatal(2, "panic: runtime error: integer divide by zero (the header names no samples)");
}

// chrom, start, end and one value per sample of every data line, on the host pool
void matrix_parse(Matrix& m) {
    const size_t R = m.rows.size(), S = m.samples.size();
    m.X.assign(R * S, 0.0);
    m.starts.assign(R, 0);
    m.ends.assign(R, 0);
    m.chrom.assign(R, {nullptr, 0});
    const int64_t per = 4096, tasks = ((int64_t)R + per - 1) / per;
    std::vector<std::string> errs((size_t)tasks);
    glhost::ThreadPool::global().run(tasks, [&](int64_t t, int) {
        for (size_t r = (size_t)t * per; r < std::min(R, (size_t)(t + 1) * per); r++) {
            const char* p = m.rows[r].p;
            const char* end = p + m.rows[r].n;
            size_t col = 0;
            auto fail = [&](const std::string& msg) { errs[(size_t)t] = "panic: line " + std::to_string(r + 1) + " of the data: " + msg; };
            for (const char* a = p;; col++) {
                const char* tab = static_cast<const char*>(memchr(a, '\t', (size_t)(end - a)));
                const char* b = tab ? tab : end;
                const char* s = a;
                if (!tab) {                                                                // only the last field is trimmed
                    while (s < b && go_space(*s)) s++;
                    while (b > s && go_space(b[-1])) b--;
                }
                if (col == 0) m.chrom[r] = {s, (size_t)(b - s)};
                else if (col < 3) {
                    int64_t v;
                    if (!dcnv_atou32(s, (size_t)(b - s), v)) { fail("strconv.Atoi: parsing \"" + std::string(s, b) + "\": invalid syntax or outside uint32"); return; }
                    (col == 1 ? m.starts[r] : m.ends[r]) = v;
                } else if (col - 3 < S) {
                    if (!dcnv_atof(s, (size_t)(b - s), m.X[r * S + col - 3])) { fail("strconv.ParseFloat: parsing \"" + std::string(s, b) + "\": invalid syntax or out of range"); return; }
                }
                if (!tab) break;
                a = tab + 1;
            }
            if (col < 2) { fail("runtime error: index out of range (fewer than 3 columns)"); return; }
            if (col + 1 != S + 3) { fail(std::to_string(col - 2) + " values but " + std::to_string(S) + " samples in the header"); return; }
        }
    });
    for (const std::string& e : errs) if (!e.empty()) fatal(2, "%s", e.c_str());
}

// The depth chart (dcnv.go:265-321 plotDepths; DESIGN §1.9) of the n x S values depth.bed holds: the reference's Chart.js
// page dd-depth-<label>.html, one stepped dataset per sample in sample order with every vertex of asValues (x = i * 16384,
// y = min(v, 2.5) as "%.2f" tokens from the GPU, written in row-block pieces made on the host pool), and dd-depth-<label>.png,
// the same lines drawn on the GPU (gl_dcnv_chart).  A file that cannot be written is reported on stderr and skipped, as
// the reference ignores plotDepths' error.
void dcnv_charts(gl_ctx* ctx, const double* X, size_t R, size_t S, const std::vector<std::string>& samples, const std::string& label) {
    const std::string png_path = "dd-depth-" + label + ".png", html_path = "dd-depth-" + label + ".html";
    const std::string xtitle = "position on " + label;
    std::vector<int64_t> first(S);
    std::vector<double> yext(2 * S), ext(4);
    std::vector<uint32_t> img((size_t)GL_PLOT_W * GL_PLOT_H);
    const char* br = getenv("GL_DCNV_CHART_BLOCK_ROWS");
    glck(ctx, gl_dcnv_chart(ctx, X, (int64_t)R, (int64_t)S, br ? atoll(br) : 0, GL_PLOT_W, GL_PLOT_H, gl_plot_line_radius((int32_t)S), first.data(),
                            yext.data(), ext.data(), img.data()), "gl_dcnv_chart");
    std::vector<uint8_t> palette(3 * (S + 1), 255);                 // draw index S - k is sample k
    for (size_t k = 0; k < S; k++) gl_plot_color((int32_t)k, 0, &palette[3 * (S - k)]);
    {
        std::vector<uint8_t> rgb((size_t)GL_PLOT_CW * GL_PLOT_CH * 3);
        if (gl_plot_compose(img.data(), palette.data(), (int32_t)(S + 1), GL_PLOT_DEPTH, ext.data(), xtitle.c_str(), "scaled coverage", rgb.data()) != GL_OK)
            fatal(1, "gl_plot_compose: %s", gl_last_error(nullptr));
        int64_t n = 0;
        gl_plot_png(rgb.data(), GL_PLOT_CW, GL_PLOT_CH, nullptr, 0, &n);
        std::vector<uint8_t> png((size_t)n);
        if (gl_plot_png(rgb.data(), GL_PLOT_CW, GL_PLOT_CH, png.data(), n, &n) != GL_OK) fatal(1, "gl_plot_png: %s", gl_last_error(nullptr));
        FILE* f = fopen(png_path.c_str(), "wb");
        bool ok = f && fwrite(png.data(), 1, (size_t)n, f) == (size_t)n;
        if (f && fclose(f) != 0) ok = false;
        if (!ok) fprintf(stderr, "dcnv: cannot write %s: %s\n", png_path.c_str(), strerror(errno));
    }
    // ---- the page
    FILE* fo = fopen(html_path.c_str(), "w");
    if (!fo) { fprintf(stderr, "dcnv: cannot write %s: %s\n", html_path.c_str(), strerror(errno)); return; }
    glhtml::Chart ch;
    ch.name = "depth"; ch.xlabel = xtitle; ch.ylabel = "scaled coverage"; ch.ymin = 0; ch.ymax = 2.5;
    std::string s = glhtml::page_open("dcnv depth " + label) + "<p><a href=\"index.html\">back to index</a></p>\n" + glhtml::chart_open(ch, 850, 550);
    fwrite(s.data(), 1, s.size(), fo);
    const size_t cols = std::max<size_t>(1, ((size_t)1 << 24) / std::max<size_t>(R, 1)), per_text = 1 << 16;
    std::vector<double> y;
    std::vector<uint8_t> tok;
    std::vector<std::string> parts;
    for (size_t k0 = 0; k0 < S; k0 += cols) {
        const size_t k1 = std::min(S, k0 + cols);
        std::vector<size_t> off(k1 - k0 + 1, 0);                     // the plotted rows of samples k0..k1, one after another
        for (size_t k = k0; k < k1; k++) off[k - k0 + 1] = off[k - k0] + (R - (size_t)first[k]);
        y.resize(off.back());
        tok.resize(off.back() * 16);
        glhost::ThreadPool::global().run((int64_t)(k1 - k0), [&](int64_t t, int) {
            const size_t k = k0 + (size_t)t;
            for (size_t i = (size_t)first[k]; i < R; i++) {
                const double v = X[i * S + k];
                y[off[t] + i - (size_t)first[k]] = v > 2.5 ? 2.5 : v;
            }
        });
        if (!y.empty()) glck(ctx, gl_format_f2(ctx, y.data(), (int64_t)y.size(), tok.data()), "gl_format_f2");
        for (size_t k = k0; k < k1; k++) {
            glhtml::Dataset ds;
            ds.label = samples[k]; ds.stepped = true; ds.width = S > 50 ? 0.2 : (S > 30 ? 0.3 : 0.4);
            gl_plot_color((int32_t)k, 0, ds.rgb);
            s = (k ? "," : "") + glhtml::dataset_head(ds);
            fwrite(s.data(), 1, s.size(), fo);
            const size_t f0 = (size_t)first[k], m = R - f0, groups = (m + per_text - 1) / per_text;
            parts.assign(groups, std::string());
            glhost::ThreadPool::global().run((int64_t)groups, [&](int64_t g, int) {
                std::string& o = parts[(size_t)g];
                o.reserve(per_text * 26);
                char num[32];
                for (size_t j = (size_t)g * per_text; j < std::min(m, ((size_t)g + 1) * per_text); j++) {
                    const size_t q = off[k - k0] + j;
                    const char* t = reinterpret_cast<const char*>(tok.data() + q * 16);
                    o += j ? ",{\"x\":" : "{\"x\":";
                    o.append(num, (size_t)snprintf(num, sizeof num, "%lld", (long long)(f0 + j) * 16384));
                    o += ",\"y\":";
                    if (!std::isfinite(y[q])) o += glhtml::num("%.2f", y[q]);                  // NaN / -Infinity, as the pages spell them
                    else if (t[0]) o.append(t, strnlen(t, 16));
                    else o += go_float("%.2f", y[q]);                                           // text longer than a token
                    o += '}';
                }
            });
            for (const std::string& p : parts) fwrite(p.data(), 1, p.size(), fo);
            fwrite("]}", 1, 2, fo);
        }
    }
    s = glhtml::chart_close(ch) + glhtml::page_close();
    fwrite(s.data(), 1, s.size(), fo);
    const bool bad = ferror(fo) != 0;
    if (fclose(fo) != 0 || bad) fprintf(stderr, "dcnv: cannot write %s: %s\n", html_path.c_str(), strerror(errno));
}

}  // namespace

static int cmd_dcnv(int argc, char** argv) {
    double svd_pct = -1;                                         // --svd PCT; < 0: off
    double chunk_w = 0;                                          // --chunk W; 0: off (the moving median of 9)
    bool noplots = false;                                        // --noplots (extension, as in indexcov): no chart files
    for (bool more = true; more && argc >= 2;) {                 // the flags, in any order, before the positionals
        more = false;
        if (strncmp(argv[1], "--chunk", 7) == 0 && (argv[1][7] == 0 || argv[1][7] == '=')) {
            ArgParser ap;
            ap.prog = "goleft dcnv";
            const int used = argv[1][7] == '=' ? 1 : 2;
            if (used == 2 && argc < 3) ap.fail("missing value for --chunk");
            const std::string v = used == 1 ? argv[1] + 8 : argv[2];
            char* endp = nullptr;
            const double w = strtod(v.c_str(), &endp);
            if (v.empty() || *endp) ap.fail("error processing chunk: strconv.ParseFloat: parsing \"" + v + "\": invalid syntax");
            if (!std::isfinite(w) || !(w > 0)) ap.fail("chunk must be a finite number > 0");
            chunk_w = w;
            more = true;
            argc -= used;
            argv += used;
        } else if (strcmp(argv[1], "--noplots") == 0) {
            noplots = more = true;
            argc -= 1;
            argv += 1;
        } else if (strncmp(argv[1], "--svd", 5) == 0 && (argv[1][5] == 0 || argv[1][5] == '=')) {
            ArgParser ap;
            ap.prog = "goleft dcnv";
            const int used = argv[1][5] == '=' ? 1 : 2;
            if (used == 2 && argc < 3) ap.fail("missing value for --svd");
            const std::string v = used == 1 ? argv[1] + 6 : argv[2];
            char* endp = nullptr;
            const double pct = strtod(v.c_str(), &endp);
            if (v.empty() || *endp) ap.fail("error processing svd: strconv.ParseFloat: parsing \"" + v + "\": invalid syntax");
            if (!std::isfinite(pct) || pct < 0) ap.fail("svd must be a finite percentage >= 0");
            svd_pct = pct;
            more = true;
            argc -= used;
            argv += used;
        }
    }
    if (argc < 3) fatal(2, "panic: runtime error: index out of range (usage: goleft dcnv <depthwed matrix> <ref.fa>)");
    const std::string path = argv[1], fasta = argv[2];
    const bool timing = getenv("GL_TIMING") != nullptr;        // phase wall clocks on stderr
    double tp = now_s();
    auto mark = [&](const char* what) { if (timing) { const double t = now_s(); fprintf(stderr, "[dcnv timing] %-22s %.3f s\n", what, t - tp); tp = t; } };
    FastaStats fa;
    fa.open(fasta);
    glhost_pool_warm();

    Matrix mx;
    matrix_read(path, mx);
    const std::vector<DcnvRow>& rows = mx.rows;
    const size_t S = mx.samples.size(), R = rows.size();
    std::string label;                                           // ivs.Chrom: set by data lines 0 and 1, so the second wins
    for (size_t r = 0; r < std::min<size_t>(R, 2); r++) {
        const void* t = memchr(rows[r].p, '\t', rows[r].n);
        if (!t) fatal(2, "panic: runtime error: slice bounds out of range [:-1] (data line %zu has no tab)", r + 1);
        label.assign(rows[r].p, (size_t)(static_cast<const char*>(t) - rows[r].p));
    }
    mark("read");

    // ---- rows on the host pool: chrom, start (clamped to 250, dcnv.go:83-85), end, S values
    matrix_parse(mx);
    std::vector<double>& X = mx.X;
    std::vector<int64_t>& starts = mx.starts;
    const std::vector<int64_t>& ends = mx.ends;
    const std::vector<std::pair<const char*, size_t>>& chrom = mx.chrom;
    for (int64_t& v : starts) v = std::max<int64_t>(v, 250);
    if (chunk_w > 0 && R < 1) fatal(2, "panic: runtime error: index out of range [0] with length 0 (no data rows)");
    if (chunk_w == 0 && R < 5) fatal(2, "panic: runtime error: index out of range (%zu data rows; the moving median needs 5)", R);
    mark("parse");

    // ---- GC of every row, a contig at a time: Faidx.Stats(chrom, start - 250, end)
    gl_ctx* ctx = open_ctx(0, "goleft dcnv");
    std::vector<double> gc(R, 0.0);
    {
        std::map<std::string, std::vector<size_t>> by_chrom;
        std::string prev;
        std::vector<size_t>* cur = nullptr;
        for (size_t r = 0; r < R; r++) {
            if (!cur || chrom[r].second != prev.size() || memcmp(chrom[r].first, prev.data(), prev.size()) != 0) {
                prev.assign(chrom[r].first, chrom[r].second);
                cur = &by_chrom[prev];
            }
            cur->push_back(r);
        }
        std::vector<int64_t> s, e;
        std::vector<double> st3;
        for (auto& kv : by_chrom) {
            const glhts::RefInfo* ri = fa.find(kv.first);
            if (!ri) { fprintf(stderr, "GC: unknown sequence %s\n", kv.first.c_str()); continue; }      // the error is printed; GC 0 (dcnv.go:86-89)
            s.clear(); e.clear();
            for (size_t r : kv.second) { s.push_back(starts[r] - 250); e.push_back(ends[r]); }
            st3.assign(s.size() * 3, 0.0);
            if (fa.stats(ctx, *ri, s, e, st3.data()))
                for (size_t k = 0; k < s.size(); k++)
                    if (e[k] < s[k] || e[k] > ri->length)
                        fatal(2, "panic: faidx: %s:%lld-%lld is outside the sequence (length %lld)", kv.first.c_str(), (long long)s[k], (long long)e[k], (long long)ri->length);
            for (size_t k = 0; k < s.size(); k++) gc[kv.second[k]] = st3[k * 3];
        }
    }
    mark("gc");
    std::vector<int64_t> inds(R);
    glck(ctx, gl_go_argsort_f64(gc.data(), (int64_t)R, inds.data()), "gl_go_argsort_f64");
    bool changed = false;
    for (size_t i = 0; i < R && !changed; i++) changed = inds[i] != (int64_t)i;
    if (!changed) go_log("WARNING: no change after sorting. This usually means .Vals is unset or same as previous run");   // debiaser.go:71-73
    mark("argsort");

    // ---- debias + normalise on the GPU, in place
    const char* bc = getenv("GL_DCNV_BLOCK_COLS");
    std::vector<double> med(S);
    if (chunk_w > 0) {                                           // the chunks over the GC values in sorted order
        std::vector<double> v(R);
        for (size_t i = 0; i < R; i++) v[i] = gc[(size_t)inds[i]];
        int64_t n_chunks = 0;
        glck(ctx, gl_dcnv_chunk_slices(v.data(), (int64_t)R, chunk_w, nullptr, 0, &n_chunks), "gl_dcnv_chunk_slices");
        std::vector<int64_t> ptr((size_t)n_chunks + 1);
        glck(ctx, gl_dcnv_chunk_slices(v.data(), (int64_t)R, chunk_w, ptr.data(), n_chunks + 1, &n_chunks), "gl_dcnv_chunk_slices");
        const int rc = gl_dcnv_normalize_chunked(ctx, X.data(), (int64_t)R, (int64_t)S, inds.data(), ptr.data(), n_chunks, 0, (int32_t)S,
                                                 bc ? atoi(bc) : 0, X.data(), (int64_t)S, med.data());
        if (rc == GL_ERANGE) fatal(2, "panic: runtime error: index out of range: %s", gl_last_error(ctx));
        glck(ctx, rc, "gl_dcnv_normalize_chunked");
        mark("normalize (chunk)");
    } else {
        const int rc = gl_dcnv_normalize(ctx, X.data(), (int64_t)R, (int64_t)S, inds.data(), 0, (int32_t)S, bc ? atoi(bc) : 0, X.data(), (int64_t)S, med.data());
        if (rc == GL_ERANGE) fatal(2, "panic: runtime error: index out of range: %s", gl_last_error(ctx));
        glck(ctx, rc, "gl_dcnv_normalize");
        mark("normalize (median 9)");
    }
    if (svd_pct >= 0) {
        std::vector<double> sv(S);
        int32_t n_removed = 0;
        glck(ctx, gl_dcnv_svd(ctx, X.data(), (int64_t)R, (int64_t)S, (int32_t)S, svd_pct, 0, sv.data(), nullptr, &n_removed, nullptr), "gl_dcnv_svd");
        double sum = 0;
        for (double v : sv) if (v > 0) sum += v;
        std::string msg = "variance:";
        for (int32_t i = 0; i < n_removed; i++) msg += " " + go_float("%.2f", 100 * sv[(size_t)i] / sum);
        go_log(msg.c_str());
        mark("svd");
    }
    if (!noplots) {                                              // plotDepths comes before depth.bed in the reference's main
        dcnv_charts(ctx, X.data(), R, S, mx.samples, label);
        mark("chart");
    }

    // ---- depth.bed: "%.2f" tokens from the GPU, rows assembled on the host pool
    FILE* fo = fopen("depth.bed", "w");
    if (!fo) fatal(2, "panic: open depth.bed: %s", strerror(errno));
    std::string head = "#chrom\tstart\tend";
    for (const std::string& s : mx.samples) head += "\t" + s;
    head += "\n";
    fwrite(head.data(), 1, head.size(), fo);
    const size_t chunk_rows = std::max<size_t>(1, ((size_t)1 << 24) / S);
    std::vector<uint8_t> tok;
    const size_t per_text = 2048;
    std::vector<std::string> parts;
    for (size_t r0 = 0; r0 < R; r0 += chunk_rows) {
        const size_t nr = std::min(chunk_rows, R - r0);
        tok.resize(nr * S * 16);
        glck(ctx, gl_format_f2(ctx, X.data() + r0 * S, (int64_t)(nr * S), tok.data()), "gl_format_f2");
        const size_t groups = (nr + per_text - 1) / per_text;
        parts.assign(groups, std::string());
        glhost::ThreadPool::global().run((int64_t)groups, [&](int64_t g, int) {
            std::string& o = parts[(size_t)g];
            char num[48];
            for (size_t r = r0 + (size_t)g * per_text; r < std::min(r0 + nr, r0 + ((size_t)g + 1) * per_text); r++) {
                o += label;
                o.append(num, (size_t)snprintf(num, sizeof num, "\t%lld\t%lld", (long long)starts[r], (long long)ends[r]));
                for (size_t c = 0; c < S; c++) {
                    const char* t = reinterpret_cast<const char*>(tok.data() + ((r - r0) * S + c) * 16);
                    o += '\t';
                    if (t[0]) o.append(t, strnlen(t, 16));
                    else o += go_float("%.2f", X[r * S + c]);                                  // text longer than a token
                }
                o += '\n';
            }
        });
        for (const std::string& p : parts) fwrite(p.data(), 1, p.size(), fo);
    }
    if (fclose(fo) != 0) fatal(1, "write depth.bed: %s", strerror(errno));
    mark("format + write");
    gl_ctx_destroy(ctx);
    return 0;
}

// ------------------------------------------------------------------------------------------------ emdepth
// emdepth/emdepth.go (a library of the reference with no command; DESIGN §1.10): `goleft emdepth [--prefix P] <matrix>` reads
// the matrix dcnv reads (matrix_read / matrix_parse; no 250 clamp, every row keeps its own chromosome), takes each value as
// float32(ParseFloat), runs the EM of every row on the GPU (gl_emdepth, row blocks sized to device memory) and walks the
// reference's Cache on the host (gl_emdepth_cnvs: Clear(nil) at every chromosome change and at the end).  Writes P.cn.bed (the
// header line, then chrom, start, end and one CN per sample) and P.cnv.bed (#chrom start end sample n cns psize: the first
// kept row's chromosome and start, the last kept row's end, the rows' CNs comma-joined).  Every error is exit 2.
static int cmd_emdepth(int argc, char** argv) {
    std::string prefix = "emdepth";
    ArgParser ap;
    ap.prog = "goleft emdepth";
    ap.add("prefix", 0, &prefix);
    ap.parse(argc, argv);
    if (ap.positional.size() != 1) fatal(2, "panic: usage: goleft emdepth [--prefix P] <matrix>");
    const bool timing = getenv("GL_TIMING") != nullptr;        // phase wall clocks on stderr
    double tp = now_s();
    auto mark = [&](const char* what) { if (timing) { const double t = now_s(); fprintf(stderr, "[emdepth timing] %-22s %.3f s\n", what, t - tp); tp = t; } };
    glhost_pool_warm();

    Matrix mx;
    matrix_read(ap.positional[0], mx);
    mark("read");
    matrix_parse(mx);
    const size_t S = mx.samples.size(), R = mx.rows.size();
    if (S == 2) fatal(2, "panic: runtime error: index out of range [2] with length 2 (median32 of 2 samples)");
    std::vector<float> X((size_t)R * S);                          // float32(strconv.ParseFloat(tok, 64))
    const int64_t per = 4096, tasks = ((int64_t)R + per - 1) / per;
    glhost::ThreadPool::global().run(tasks, [&](int64_t t, int) {
        for (size_t i = (size_t)t * per * S; i < std::min(R, (size_t)(t + 1) * per) * S; i++) X[i] = (float)mx.X[i];
    });
    mark("parse");

    gl_ctx* ctx = open_ctx(0, "goleft emdepth");
    std::vector<uint8_t> cells((size_t)R * S);
    const char* br = getenv("GL_EMDEPTH_BLOCK_ROWS");
    const int rc = gl_emdepth(ctx, X.data(), (int64_t)R, (int64_t)S, (int32_t)S, br ? atoll(br) : 0, cells.data(), nullptr);
    if (rc == GL_EINVAL) fatal(2, "panic: %s", gl_last_error(ctx));
    glck(ctx, rc, "gl_emdepth");
    int64_t n_unc = 0;
    gl_emdepth_stats(ctx, nullptr, &n_unc, nullptr);
    if (n_unc) fprintf(stderr, "emdepth: %lld cells were decided inside the error band of the reference's CPU-dependent Exp / Log\n", (long long)n_unc);
    mark("em");

    const std::string cn_path = prefix + ".cn.bed", cnv_path = prefix + ".cnv.bed";
    FILE* fo = fopen(cn_path.c_str(), "w");
    if (!fo) fatal(2, "panic: open %s: %s", cn_path.c_str(), strerror(errno));
    std::string head;
    for (size_t i = 0; i < mx.header.size(); i++) head += (i ? "\t" : "") + mx.header[i];
    head += "\n";
    fwrite(head.data(), 1, head.size(), fo);
    const size_t per_text = 4096, groups = (R + per_text - 1) / per_text, group_batch = 64;
    for (size_t g0 = 0; g0 < groups; g0 += group_batch) {
        const size_t ng = std::min(group_batch, groups - g0);
        std::vector<std::string> parts(ng);
        glhost::ThreadPool::global().run((int64_t)ng, [&](int64_t k, int) {
            std::string& o = parts[(size_t)k];
            char num[48];
            const size_t r0 = (g0 + (size_t)k) * per_text;
            for (size_t r = r0; r < std::min(R, r0 + per_text); r++) {
                o.append(mx.chrom[r].first, mx.chrom[r].second);
                o.append(num, (size_t)snprintf(num, sizeof num, "\t%lld\t%lld", (long long)mx.starts[r], (long long)mx.ends[r]));
                for (size_t c = 0; c < S; c++) {
                    o += '\t';
                    o += (char)('0' + (cells[r * S + c] & 15));
                }
                o += '\n';
            }
        });
        for (const std::string& p : parts) fwrite(p.data(), 1, p.size(), fo);
    }
    if (fclose(fo) != 0) fatal(1, "write %s: %s", cn_path.c_str(), strerror(errno));
    mark("cn.bed");

    std::vector<int64_t> breaks;                                  // rows where a chromosome starts
    for (size_t r = 1; r < R; r++)
        if (mx.chrom[r].second != mx.chrom[r - 1].second || memcmp(mx.chrom[r].first, mx.chrom[r - 1].first, mx.chrom[r].second) != 0)
            breaks.push_back((int64_t)r);
    int64_t nc = 0, nr = 0;
    auto walk = [&](int32_t* smp, int32_t* psz, int64_t* ptr, int64_t* rows) {
        return gl_emdepth_cnvs(cells.data(), (int64_t)R, (int32_t)S, mx.starts.data(), mx.ends.data(), breaks.data(), (int64_t)breaks.size(),
                               smp, psz, ptr, nc, &nc, rows, nr, &nr);
    };
    if (walk(nullptr, nullptr, nullptr, nullptr) != GL_OK) fatal(1, "gl_emdepth_cnvs: bad arguments");
    std::vector<int32_t> smp((size_t)nc), psz((size_t)nc);
    std::vector<int64_t> ptr((size_t)nc + 1), rows((size_t)nr);
    if (walk(smp.data(), psz.data(), ptr.data(), rows.data()) != GL_OK) fatal(1, "gl_emdepth_cnvs: bad arguments");
    fo = fopen(cnv_path.c_str(), "w");
    if (!fo) fatal(2, "panic: open %s: %s", cnv_path.c_str(), strerror(errno));
    std::string o = "#chrom\tstart\tend\tsample\tn\tcns\tpsize\n";
    char num[64];
    for (int64_t i = 0; i < nc; i++) {
        const int64_t a = rows[(size_t)ptr[(size_t)i]], b = rows[(size_t)ptr[(size_t)i + 1] - 1];
        o.append(mx.chrom[(size_t)a].first, mx.chrom[(size_t)a].second);
        o.append(num, (size_t)snprintf(num, sizeof num, "\t%lld\t%lld\t", (long long)mx.starts[(size_t)a], (long long)mx.ends[(size_t)b]));
        o += mx.samples[(size_t)smp[(size_t)i]];
        o.append(num, (size_t)snprintf(num, sizeof num, "\t%lld\t", (long long)(ptr[(size_t)i + 1] - ptr[(size_t)i])));
        for (int64_t k = ptr[(size_t)i]; k < ptr[(size_t)i + 1]; k++) {
            if (k > ptr[(size_t)i]) o += ',';
            o += (char)('0' + (cells[(size_t)rows[(size_t)k] * S + (size_t)smp[(size_t)i]] & 15));
        }
        o.append(num, (size_t)snprintf(num, sizeof num, "\t%d\n", psz[(size_t)i]));
    }
    fwrite(o.data(), 1, o.size(), fo);
    if (fclose(fo) != 0) fatal(1, "write %s: %s", cnv_path.c_str(), strerror(errno));
    mark("cnv.bed");
    gl_ctx_destroy(ctx);
    return 0;
}

// ------------------------------------------------------------------------------------------------ cnveval
// cnveval/cmd/cnveval/cnveval.go (a separate binary of the reference; DESIGN §1.12): `goleft cnveval [-m|--minoverlap 0.4]
// [-s|--limitsamples] truth.bed test.bed` scores the test set's CNV calls against the truth set and prints precision and
// recall per size class.  Both files are chrom, start, end, CN and comma-separated samples (a test line uses its first
// sample), read whole (plain, gzip or "-"); ReadString('\n') drops a final line without "\n"; lines starting with '#' are
// skipped.  The counts come from gl_cnveval on the GPU.  Argument errors exit 255 (go-arg), the reference's panics exit 2.
// Unlike the reference, no x.cpu.pprof profile is written into the working directory.
namespace {

struct CnvLine { std::string chrom; int64_t start, end, cn; std::vector<std::string> samples; };

// strconv.Atoi: optional sign, decimal digits, int64 range
bool go_atoi(const std::string& t, int64_t& v) {
    size_t k = 0;
    const bool neg = !t.empty() && t[0] == '-';
    if (!t.empty() && (t[0] == '+' || t[0] == '-')) k = 1;
    if (k == t.size()) return false;
    unsigned long long u = 0;
    for (; k < t.size(); k++) {
        if (t[k] < '0' || t[k] > '9') return false;
        const unsigned d = (unsigned)(t[k] - '0');
        if (u > (~0ull - d) / 10) return false;
        u = u * 10 + d;
    }
    if (neg ? u > (1ull << 63) : u > (1ull << 63) - 1) return false;
    v = neg ? (int64_t)(0 - u) : (int64_t)u;
    return true;
}

std::vector<std::string> split(const std::string& s, char sep) {
    std::vector<std::string> out;
    for (size_t a = 0;;) {
        const size_t b = s.find(sep, a);
        if (b == std::string::npos) { out.push_back(s.substr(a)); return out; }
        out.push_back(s.substr(a, b - a));
        a = b + 1;
    }
}

// parseTruth (cnveval.go:65-107); samples (non-null): keep a line only when one of its samples is in the set
std::vector<CnvLine> cnv_parse(const std::string& path, const std::map<std::string, int>* samples) {
    const std::string text = read_whole(path);
    std::vector<CnvLine> out;
    for (size_t a = 0; a < text.size();) {
        const size_t nl = text.find('\n', a);
        if (nl == std::string::npos) break;
        std::string line = text.substr(a, nl - a);
        a = nl + 1;
        if (line.empty() || line[0] != '#') {
            while (!line.empty() && (line.back() == '\r' || line.back() == '\n')) line.pop_back();   // TrimRight(l, "\r\n")
            std::vector<std::string> f = split(line, '\t');
            if (f.size() < 5) fatal(2, "panic: expected five fields for CNVs");
            CnvLine c;
            c.chrom = f[0];
            for (int k = 1; k <= 3; k++)
                if (!go_atoi(f[(size_t)k], k == 1 ? c.start : (k == 2 ? c.end : c.cn)))
                    fatal(2, "panic: strconv.Atoi: parsing \"%s\": invalid syntax or value out of range", f[(size_t)k].c_str());
            c.samples = split(f[4], ',');
            if (samples) {
                bool found = false;
                for (const std::string& s : c.samples) found = found || samples->count(s);
                if (!found) continue;
            }
            out.push_back(std::move(c));
        }
    }
    return out;
}

}  // namespace

static int cmd_cnveval(int argc, char** argv) {
    std::string m = "0.4";
    bool limit = false;
    ArgParser ap;
    ap.prog = "cnveval";
    ap.add("minoverlap", 'm', &m);
    ap.addb("limitsamples", 's', &limit);
    ap.parse(argc, argv);
    if (ap.positional.size() < 2) ap.fail(ap.positional.empty() ? "truth is required" : "test is required");
    if (ap.positional.size() > 2) ap.fail("too many positional arguments at '" + ap.positional[2] + "'");
    char* endp = nullptr;
    const double po = strtod(m.c_str(), &endp);
    if (m.empty() || *endp) ap.fail("error processing minoverlap: strconv.ParseFloat: parsing \"" + m + "\": invalid syntax");
    if (po > 1 || po <= 0) ap.fail("minoverlap must be between 0 and 1");              // NaN passes, as in the reference
    const bool timing = getenv("GL_TIMING") != nullptr;        // phase wall clocks on stderr
    double tp = now_s();
    auto mark = [&](const char* what) { if (timing) { const double t = now_s(); fprintf(stderr, "[cnveval timing] %-22s %.3f s\n", what, t - tp); tp = t; } };

    const std::vector<CnvLine> tests = cnv_parse(ap.positional[1], nullptr);
    char msg[128];
    snprintf(msg, sizeof msg, "cnvs in test-set (%zu)", tests.size());
    go_log(msg);
    std::map<std::string, int> first;                            // -s: the first sample of every test line
    for (const CnvLine& c : tests) first.emplace(c.samples[0], 0);
    const std::vector<CnvLine> truths = cnv_parse(ap.positional[0], limit ? &first : nullptr);
    size_t n_mem = 0;
    for (const CnvLine& t : truths) n_mem += t.samples.size();
    snprintf(msg, sizeof msg, "%zu total cnvs in truth-set (%zu)", n_mem, truths.size());
    go_log(msg);
    mark("read + parse");

    // chrom ranks in bytewise name order; samples numbered as met
    std::map<std::string, int32_t> chrom;
    for (const CnvLine& c : tests) chrom.emplace(c.chrom, 0);
    for (const CnvLine& t : truths) chrom.emplace(t.chrom, 0);
    int32_t r = 0;
    for (auto& kv : chrom) kv.second = r++;
    std::map<std::string, int32_t> sample;
    auto sid = [&](const std::string& s) { return sample.emplace(s, (int32_t)sample.size()).first->second; };
    std::vector<int32_t> c_sample, c_chrom, t_chrom, t_mem_sample;
    std::vector<int64_t> c_start, c_end, c_cn, t_start, t_end, t_cn, t_mem_ptr{0};
    for (const CnvLine& c : tests) {
        c_sample.push_back(sid(c.samples[0])); c_chrom.push_back(chrom[c.chrom]);
        c_start.push_back(c.start); c_end.push_back(c.end); c_cn.push_back(c.cn);
    }
    for (const CnvLine& t : truths) {
        t_chrom.push_back(chrom[t.chrom]); t_start.push_back(t.start); t_end.push_back(t.end); t_cn.push_back(t.cn);
        for (const std::string& s : t.samples) t_mem_sample.push_back(sid(s));
        t_mem_ptr.push_back((int64_t)t_mem_sample.size());
    }
    const int32_t S = (int32_t)sample.size();
    mark("intern");

    gl_ctx* ctx = open_ctx(0, "goleft cnveval");
    std::vector<uint64_t> st((size_t)S * 12);
    const int rc = gl_cnveval(ctx, S, c_sample.data(), c_chrom.data(), c_start.data(), c_end.data(), c_cn.data(), (int64_t)tests.size(),
                              t_chrom.data(), t_start.data(), t_end.data(), t_cn.data(), (int64_t)truths.size(), t_mem_ptr.data(),
                              t_mem_sample.data(), po, st.data());
    if (rc == GL_EINVAL) fatal(2, "panic: %s (calls count test-set lines, truths truth-set lines, from 0, without '#' lines)", gl_last_error(ctx));
    glck(ctx, rc, "gl_cnveval");
    mark("evaluate");

    uint64_t tab[4][4] = {};                                      // Tabulate (cnveval.go:118-133)
    for (int32_t s = 0; s < S; s++)
        for (int c = 0; c < 3; c++)
            for (int k = 0; k < 4; k++) tab[c][k] += st[(size_t)s * 12 + (size_t)c * 4 + (size_t)k];
    for (int c = 0; c < 3; c++)
        for (int k = 0; k < 4; k++) tab[3][k] += tab[c][k];
    static const char* kClass[4] = {"0-20000", "20000-100000", ">=100000", "all"};
    for (int c = 0; c < 4; c++) {
        const long long TP = (long long)tab[c][0], FP = (long long)tab[c][1], FN = (long long)tab[c][2];
        const std::string p = go_float("%.4f", (double)TP / (double)(TP + FP)), q = go_float("%.4f", (double)TP / (double)(TP + FN));
        // Stat.String's "%-04d": with '-', Go and C both ignore '0' and pad with spaces on the right
        printf("size-class: %-12s | precision: %s (%-4lld / (%-4lld + %-4lld)) recall: %s (%-4lld / (%-4lld + %-4lld))\n",
               kClass[c], p.c_str(), TP, TP, FP, q.c_str(), TP, TP, FN);
    }
    mark("tabulate + print");
    gl_ctx_destroy(ctx);
    return 0;
}

static void print_progs() {                                                          // cmd/goleft/goleft.go:33-53
    fprintf(stderr, "goleft Version: %s (GPU engine: %s)\n\n", kVersion, gl_version());
    fprintf(stderr, "covstats    : coverage and insert-size statistics on bams by sampling\n");
    fprintf(stderr, "depth       : parallelize calls to samtools in user-defined windows\n");
    fprintf(stderr, "depthwed    : matricize output from depth to n-sites * n-samples\n");
    fprintf(stderr, "indexcov    : quick coverage estimate using only the bam index\n");
    fprintf(stderr, "indexsplit  : create regions of even coverage across bams/crams\n");
    fprintf(stderr, "samplename  : report samplename(s) from a bam's SM tag\n");
    fprintf(stderr, "multidepth  : (extension; a separate binary in goleft) blocks of sufficient coverage across many bams\n");
    fprintf(stderr, "dcnv        : (extension; a separate binary in goleft) GC-debias and median-normalise a depthwed matrix\n");
    fprintf(stderr, "emdepth     : (extension; a library in goleft) per-sample copy numbers and CNVs from a depth matrix\n");
    fprintf(stderr, "cnveval     : (extension; a separate binary in goleft) precision and recall of CNV calls against a truth set\n");
}

int main(int argc, char** argv) {
    if (argc < 2) { print_progs(); return 0; }
    const std::string prog = argv[1];
    if (prog == "depth") return cmd_depth(argc - 1, argv + 1);
    if (prog == "indexcov") return cmd_indexcov(argc - 1, argv + 1);
    if (prog == "covstats") return cmd_covstats(argc - 1, argv + 1);
    if (prog == "depthwed") return cmd_depthwed(argc - 1, argv + 1);
    if (prog == "indexsplit") return cmd_indexsplit(argc - 1, argv + 1);
    if (prog == "samplename") return cmd_samplename(argc - 1, argv + 1);
    if (prog == "multidepth") return cmd_multidepth(argc - 1, argv + 1);
    if (prog == "dcnv") return cmd_dcnv(argc - 1, argv + 1);
    if (prog == "emdepth") return cmd_emdepth(argc - 1, argv + 1);
    if (prog == "cnveval") return cmd_cnveval(argc - 1, argv + 1);
    print_progs();
    return 1;
}
