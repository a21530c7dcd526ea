// Microbenchmark: throughput of shared-memory atomicAdd (spread addresses inside a 4096-int tile)
// vs global red.add on an L2-resident vs HBM-sized array.  Informs the depth scatter design.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#define CK(x) do{cudaError_t e=(x); if(e!=cudaSuccess){printf("%s: %s\n",#x,cudaGetErrorString(e)); return 1;}}while(0)

__device__ __forceinline__ unsigned hash32(unsigned x){ x^=x>>16; x*=0x7feb352dU; x^=x>>15; x*=0x846ca68bU; x^=x>>16; return x; }

template<int MODE>  // 0: random spread, 1: sorted-like (addresses within +-8 of 6*i)
__global__ void smem_atomics(int* out, int iters){
    __shared__ int tile[4097];
    for(int i=threadIdx.x;i<4097;i+=blockDim.x) tile[i]=0;
    __syncthreads();
    unsigned h = hash32(blockIdx.x*blockDim.x+threadIdx.x+1);
    for(int it=0; it<iters; it++){
        unsigned a;
        if (MODE==0) { h = hash32(h); a = h & 4095; }
        else { a = ((it*blockDim.x + threadIdx.x)*6u + (hash32(h+it)&7)) & 4095; }
        atomicAdd(&tile[a], 1);
        atomicAdd(&tile[(a+150)&4095], -1);
    }
    __syncthreads();
    int s=0; for(int i=threadIdx.x;i<4096;i+=blockDim.x) s+=tile[i];
    if (s==123456789) out[0]=s;
}

__global__ void global_reds(int* arr, unsigned mask, long long n_per_thread){
    // sorted-like: thread i touches positions ~6*i (+ jitter) and +150
    unsigned long long gid = (unsigned long long)blockIdx.x*blockDim.x+threadIdx.x;
    unsigned long long nthreads = (unsigned long long)gridDim.x*blockDim.x;
    for(long long k=0;k<n_per_thread;k++){
        unsigned long long i = k*nthreads + gid;
        unsigned a = (unsigned)((i*6 + (hash32((unsigned)i)&7)) & mask);
        atomicAdd(arr + a, 1);
        atomicAdd(arr + ((a+150)&mask), -1);
    }
}

int main(){
    int* out; CK(cudaMalloc(&out, 4));
    cudaEvent_t e0,e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    int sms, khz; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0)); CK(cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0));
    const double ghz = khz / 1e6;
    int iters=2048; int grid=sms*8;
    for(int mode=0; mode<2; mode++){
        for(int rep=0;rep<3;rep++){
            cudaEventRecord(e0);
            if(mode==0) smem_atomics<0><<<grid,256>>>(out,iters); else smem_atomics<1><<<grid,256>>>(out,iters);
            cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
            float ms; cudaEventElapsedTime(&ms,e0,e1);
            double n = 2.0*grid*256.0*iters;
            if(rep==2) printf("smem atomics mode %d: %.1f G atomics/s (%.3f ms), per SM per clk @%.2fGHz: %.2f\n", mode, n/ms/1e6, ms, ghz, n/ms/1e6/sms/ghz);
        }
    }
    for(int lg=22; lg<=27; lg+=5){   // 16 MB (L2 resident) and 512 MB (HBM)
        size_t n = (size_t)1<<lg; int* arr; CK(cudaMalloc(&arr, n*4)); CK(cudaMemset(arr,0,n*4));
        for(int rep=0;rep<3;rep++){
            cudaEventRecord(e0);
            global_reds<<<sms*16,256>>>(arr,(unsigned)(n-1), 16);
            cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
            float ms; cudaEventElapsedTime(&ms,e0,e1);
            double cnt = 2.0*sms*16*256*16;
            if(rep==2) printf("global reds on %zu MB array: %.1f G reds/s (%.3f ms)\n", n*4>>20, cnt/ms/1e6, ms);
        }
        cudaFree(arr);
    }
    return 0;
}
