// gl_ctx.cu — context lifetime, device/pinned memory plumbing, timers.
#include "gl_common.cuh"
#include <stdarg.h>
#include <string.h>
#include <ctype.h>
#include <sched.h>

thread_local std::string g_gl_err;

int gl_fail(gl_ctx* ctx, int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_gl_err = buf;
    if (ctx) ctx->err = buf;
    return code;
}

int gl_buf_reserve(gl_ctx* ctx, gl_buf& b, size_t bytes) {
    if (bytes <= b.cap) return GL_OK;
    if (b.p) {
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        GL_CUDA(ctx, cudaFree(b.p));
        b.p = nullptr;
        b.cap = 0;
    }
    size_t want = (bytes + 255) & ~size_t(255);
    cudaError_t e = cudaMalloc(&b.p, want);
    if (e != cudaSuccess) {
        b.p = nullptr;
        cudaGetLastError();
        return gl_fail(ctx, GL_ENOMEM, "cudaMalloc(%zu bytes): %s", want, cudaGetErrorString(e));
    }
    b.cap = want;
    return GL_OK;
}

int gl_pinned_reserve(gl_ctx* ctx, size_t bytes, size_t want) {
    if (ctx->pack_pinned_bytes >= bytes) return GL_OK;
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream));
    if (ctx->pack_pinned) cudaFreeHost(ctx->pack_pinned);
    ctx->pack_pinned = nullptr;
    ctx->pack_pinned_bytes = 0;
    cudaError_t e = cudaHostAlloc(&ctx->pack_pinned, want, cudaHostAllocDefault);
    if (e != cudaSuccess) {
        ctx->pack_pinned = nullptr;
        cudaGetLastError();
        return gl_fail(ctx, GL_ENOMEM, "cudaHostAlloc(%zu): %s", want, cudaGetErrorString(e));
    }
    ctx->pack_pinned_bytes = want;
    return GL_OK;
}

static void buf_free(gl_buf& b) {
    if (b.p) cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
}

extern "C" {

const char* gl_version(void) { return "goleft_b200 0.1.0 sm_90a"; }

int gl_device_count(int* n) {
    if (!n) return gl_fail(nullptr, GL_EINVAL, "null out pointer");
    int c = 0;
    cudaError_t e = cudaGetDeviceCount(&c);
    if (e != cudaSuccess) {
        *n = 0;
        cudaGetLastError();
        return gl_fail(nullptr, GL_ECUDA, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
    }
    *n = c;
    return GL_OK;
}

int gl_ctx_create(int device, gl_ctx** out) {
    if (!out) return gl_fail(nullptr, GL_EINVAL, "null out pointer");
    *out = nullptr;
    int n = 0;
    GL_CHECK(gl_device_count(&n));
    if (n <= 0) return gl_fail(nullptr, GL_ECUDA, "no CUDA device visible: libgoleft_b200 has no CPU fallback");
    if (device < 0 || device >= n) return gl_fail(nullptr, GL_EINVAL, "device %d out of range [0,%d)", device, n);
    gl_ctx* ctx = new gl_ctx();
    ctx->device = device;
    cudaError_t e = cudaSetDevice(device);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->d2h_stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreate(&ctx->ev0);
    if (e == cudaSuccess) e = cudaEventCreate(&ctx->ev1);
    for (int i = 0; i < 2 && e == cudaSuccess; i++) {
        e = cudaEventCreateWithFlags(&ctx->ev_copy[i], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->ev_used[i], cudaEventDisableTiming);
    }
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->ev_hdr, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaHostAlloc(reinterpret_cast<void**>(&ctx->hdr_host), 4 * sizeof(uint64_t), cudaHostAllocMapped);
    if (e == cudaSuccess) e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&ctx->hdr_dev), ctx->hdr_host, 0);
    if (e == cudaSuccess) {
        cudaDeviceProp prop;
        e = cudaGetDeviceProperties(&prop, device);
        if (e == cudaSuccess) {
            ctx->sm_count = prop.multiProcessorCount;
            if (prop.major != 9 || prop.minor != 0) {   // sm_90a SASS only, no PTX: nothing else can load it
                int rc = gl_fail(nullptr, GL_ECUDA, "device %d is sm_%d%d; this library is built for sm_90a only",
                                 device, prop.major, prop.minor);
                delete ctx;
                return rc;
            }
        }
    }
    if (e != cudaSuccess) {
        int rc = gl_fail(nullptr, GL_ECUDA, "gl_ctx_create: %s", cudaGetErrorString(e));
        delete ctx;
        return rc;
    }
    *out = ctx;
    return GL_OK;
}

// Pin the calling thread (and the threads it creates afterwards: the library's pool, a feeder) to the CPUs of the NUMA
// node the GPU hangs off, so pinned staging buffers are first-touched next to the GPU's PCIe root and H2D copies do not
// cross the socket link (round 1: 8 ranks on one box, the ranks on the far socket lost a third of their H2D bandwidth).
// share_index/share_count split that node's CPUs between the ranks that share it.  Best effort: *node = -1 when the
// topology cannot be read (then nothing is changed).
int gl_device_numa_node(int device, int* node) {
    if (!node) return gl_fail(nullptr, GL_EINVAL, "null out pointer");
    *node = -1;
    char bus[64] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) { cudaGetLastError(); return gl_fail(nullptr, GL_ECUDA, "cudaDeviceGetPCIBusId(%d) failed", device); }
    for (char* c = bus; *c; c++) *c = (char)tolower((unsigned char)*c);
    char path[256];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r");
    int nd = -1;
    if (f) { if (fscanf(f, "%d", &nd) != 1) nd = -1; fclose(f); }
    *node = nd;
    return GL_OK;
}

int gl_bind_numa_for_device(int device, int share_index, int share_count, int* node, int* n_cpus) {
    if (node) *node = -1;
    if (n_cpus) *n_cpus = 0;
    int nd = -1;
    GL_CHECK(gl_device_numa_node(device, &nd));
    if (nd < 0) return GL_OK;
    char path[256];
    FILE* f;
    snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", nd);
    f = fopen(path, "r");
    if (!f) return GL_OK;
    char list[4096] = {0};
    if (!fgets(list, sizeof list, f)) list[0] = 0;
    fclose(f);
    std::vector<int> cpus;
    for (char* p = list; *p;) {
        char* e = nullptr;
        long a = strtol(p, &e, 10);
        if (e == p) break;
        long b = a;
        if (*e == '-') { p = e + 1; b = strtol(p, &e, 10); }
        for (long c = a; c <= b && c < CPU_SETSIZE; c++) cpus.push_back((int)c);
        p = (*e == ',') ? e + 1 : e;
        if (*e != ',') break;
    }
    if (cpus.empty()) return GL_OK;
    // hyper-thread siblings sit in the second half of the list (0-31,64-95): deal whole cores, both siblings together
    std::vector<int> mine;
    if (share_count > 1 && share_index >= 0 && share_index < share_count) {
        const size_t half = cpus.size() / 2;
        const bool paired = cpus.size() % 2 == 0 && half > 0;
        const size_t cores = paired ? half : cpus.size();
        const size_t lo = cores * (size_t)share_index / (size_t)share_count, hi = cores * (size_t)(share_index + 1) / (size_t)share_count;
        for (size_t k = lo; k < hi; k++) { mine.push_back(cpus[k]); if (paired) mine.push_back(cpus[half + k]); }
    }
    if (mine.empty()) mine = cpus;
    cpu_set_t set;
    CPU_ZERO(&set);
    for (int c : mine) CPU_SET(c, &set);
    if (sched_setaffinity(0, sizeof set, &set) != 0) return GL_OK;
    if (node) *node = nd;
    if (n_cpus) *n_cpus = (int)mine.size();
    return GL_OK;
}

int gl_comm_destroy(gl_ctx* ctx);

int gl_ctx_destroy(gl_ctx* ctx) {
    if (!ctx) return GL_OK;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    if (ctx->nccl) gl_comm_destroy(ctx);
    md_free(ctx);
    cs_free(ctx);
    buf_free(ctx->diff); buf_free(ctx->win_min);
    buf_free(ctx->run_start); buf_free(ctx->run_class); buf_free(ctx->scratch);
    buf_free(ctx->run_tmp_start); buf_free(ctx->run_tmp_class);
    buf_free(ctx->store_s); buf_free(ctx->store_e); buf_free(ctx->packed);
    buf_free(ctx->flush); buf_free(ctx->misc); buf_free(ctx->fasta);
    buf_free(ctx->bam_comp); buf_free(ctx->bam_out); buf_free(ctx->bam_seg);
    buf_free(ctx->text_slots); buf_free(ctx->text_blk); buf_free(ctx->text_len); buf_free(ctx->text_out[0]); buf_free(ctx->text_out[1]);
    for (int i = 0; i < 2; i++) {
        if (ctx->pinned[i]) cudaFreeHost(ctx->pinned[i]);
        if (ctx->ev_copy[i]) cudaEventDestroy(ctx->ev_copy[i]);
        if (ctx->ev_used[i]) cudaEventDestroy(ctx->ev_used[i]);
    }
    if (ctx->pack_pinned) cudaFreeHost(ctx->pack_pinned);
    if (ctx->hdr_host) cudaFreeHost(ctx->hdr_host);
    if (ctx->ev_hdr) cudaEventDestroy(ctx->ev_hdr);
    free(ctx->esc_buf);
    for (auto& r : ctx->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    for (auto e : ctx->prof_pool) cudaEventDestroy(e);
    for (auto e : ctx->ev_chunk) cudaEventDestroy(e);
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->d2h_stream) cudaStreamDestroy(ctx->d2h_stream);
    if (ctx->comm_stream) cudaStreamDestroy(ctx->comm_stream);
    if (ctx->ev_comm) cudaEventDestroy(ctx->ev_comm);
    delete ctx;
    return GL_OK;
}

const char* gl_last_error(gl_ctx* ctx) { return ctx ? ctx->err.c_str() : g_gl_err.c_str(); }

int gl_sync(gl_ctx* ctx) {
    GL_CHECK(gl_use(ctx));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_launch_count(gl_ctx* ctx, int64_t* n) {
    if (!ctx || !n) return gl_fail(ctx, GL_EINVAL, "null argument");
    *n = ctx->launches;
    return GL_OK;
}

int gl_stream_handle(gl_ctx* ctx, uint64_t* stream) {
    if (!ctx || !stream) return gl_fail(ctx, GL_EINVAL, "null argument");
    *stream = (uint64_t)(uintptr_t)ctx->stream;
    return GL_OK;
}

int gl_dev_alloc(gl_ctx* ctx, int64_t bytes, void** d_ptr) {
    GL_CHECK(gl_use(ctx));
    if (!d_ptr || bytes < 0) return gl_fail(ctx, GL_EINVAL, "gl_dev_alloc: bad argument");
    *d_ptr = nullptr;
    cudaError_t e = cudaMalloc(d_ptr, (size_t)(bytes > 0 ? bytes : 1));
    if (e != cudaSuccess) {
        cudaGetLastError();
        return gl_fail(ctx, GL_ENOMEM, "cudaMalloc(%lld): %s", (long long)bytes, cudaGetErrorString(e));
    }
    return GL_OK;
}

int gl_dev_free(gl_ctx* ctx, void* d_ptr) {
    GL_CHECK(gl_use(ctx));
    if (d_ptr) GL_CUDA(ctx, cudaFree(d_ptr));
    return GL_OK;
}

int gl_host_alloc_pinned(gl_ctx* ctx, int64_t bytes, void** h_ptr) {
    GL_CHECK(gl_use(ctx));
    if (!h_ptr || bytes < 0) return gl_fail(ctx, GL_EINVAL, "gl_host_alloc_pinned: bad argument");
    *h_ptr = nullptr;
    cudaError_t e = cudaHostAlloc(h_ptr, (size_t)(bytes > 0 ? bytes : 1), cudaHostAllocDefault);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return gl_fail(ctx, GL_ENOMEM, "cudaHostAlloc(%lld): %s", (long long)bytes, cudaGetErrorString(e));
    }
    return GL_OK;
}

int gl_host_free_pinned(gl_ctx* ctx, void* h_ptr) {
    GL_CHECK(gl_use(ctx));
    if (h_ptr) GL_CUDA(ctx, cudaFreeHost(h_ptr));
    return GL_OK;
}

int gl_memcpy_h2d(gl_ctx* ctx, void* d_dst, const void* h_src, int64_t bytes) {
    GL_CHECK(gl_use(ctx));
    if (bytes < 0) return gl_fail(ctx, GL_EINVAL, "negative size");
    if (bytes == 0) return GL_OK;
    GL_CUDA(ctx, cudaMemcpyAsync(d_dst, h_src, (size_t)bytes, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_memcpy_d2h(gl_ctx* ctx, void* h_dst, const void* d_src, int64_t bytes) {
    GL_CHECK(gl_use(ctx));
    if (bytes < 0) return gl_fail(ctx, GL_EINVAL, "negative size");
    if (bytes == 0) return GL_OK;
    GL_CUDA(ctx, cudaMemcpyAsync(h_dst, d_src, (size_t)bytes, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_timer_start(gl_ctx* ctx) {
    GL_CHECK(gl_use(ctx));
    GL_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
    return GL_OK;
}

int gl_timer_stop_ms(gl_ctx* ctx, float* ms) {
    GL_CHECK(gl_use(ctx));
    if (!ms) return gl_fail(ctx, GL_EINVAL, "null out pointer");
    GL_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
    GL_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
    GL_CUDA(ctx, cudaEventElapsedTime(ms, ctx->ev0, ctx->ev1));
    return GL_OK;
}

int gl_profile_enable(gl_ctx* ctx, int on) {
    GL_CHECK(gl_use(ctx));
    ctx->prof_on = on != 0;
    return GL_OK;
}

// "name ms\n" per kernel launched since the last read; synchronizes the stream
int gl_profile_read(gl_ctx* ctx, char* buf, int64_t cap, int64_t* needed) {
    GL_CHECK(gl_use(ctx));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::string out;
    for (auto& r : ctx->prof) {
        float ms = 0;
        cudaEventElapsedTime(&ms, r.a, r.b);
        char line[128];
        snprintf(line, sizeof line, "%s %.6f\n", r.name, ms);
        out += line;
        ctx->prof_pool.push_back(r.a);
        ctx->prof_pool.push_back(r.b);
    }
    ctx->prof.clear();
    if (needed) *needed = (int64_t)out.size() + 1;
    if (buf && cap > 0) {
        size_t n = std::min<size_t>(out.size(), (size_t)cap - 1);
        memcpy(buf, out.data(), n);
        buf[n] = 0;
    }
    return GL_OK;
}

int gl_flush_l2(gl_ctx* ctx) {
    GL_CHECK(gl_use(ctx));
    const size_t bytes = size_t(256) << 20;   // 256 MiB > 50 MB L2
    GL_CHECK(gl_buf_reserve(ctx, ctx->flush, bytes));
    GL_CUDA(ctx, cudaMemsetAsync(ctx->flush.p, 0x5a, bytes, ctx->stream));
    return GL_OK;
}

}  // extern "C"
