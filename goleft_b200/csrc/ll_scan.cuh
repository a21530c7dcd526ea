// ll_scan.cuh — the one-CTA scan that places units (bamgpu.cu, covstats.cu).
#pragma once

// exclusive scan of n long longs, one CTA (n = the units of one reference or the record blocks of one covstats batch: thousands)
static __global__ void __launch_bounds__(1024) ll_scan_kernel(const long long* __restrict__ in, long long* __restrict__ out, int n) {
    __shared__ long long s_w[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int per = (n + 1 + 1023) / 1024;
    const int b = tid * per, e = min(n + 1, b + per);
    long long loc = 0;
    for (int i = b; i < e; i++) loc += i < n ? in[i] : 0;
    long long inc = loc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const long long y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) s_w[warp] = inc;
    __syncthreads();
    long long run = inc - loc;
    for (int k = 0; k < warp; k++) run += s_w[k];
    for (int i = b; i < e; i++) { out[i] = run; run += i < n ? in[i] : 0; }
}
