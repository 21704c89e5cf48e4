// Dev micro-benchmark: one PAIR step of the capacity-1 slot-0 chain (two topics from one counter snapshot) against one
// level of the one-topic loop, in the same run, at 128 and 256 threads.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pair_floor pair_floor.cu && ./pair_floor
// level: 16-byte record read, 3 counter reads, decide, counter store, 16-byte global store, bar.sync.
// pair:  2 + 3 16-byte record reads (p, q, q's holders), 15 independent counter reads, a decide two levels deep, bar.sync,
//        2 shared-memory adds, 2 16-byte global stores, bar.sync.
// The pair step pays if it costs clearly less than two levels (the gate: below 1.5 levels).
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ int ld(const int* c, uint32_t a) {
    int v;
    asm volatile("ld.volatile.shared.s32 %0, [%1];" : "=r"(v) : "r"((uint32_t)__cvta_generic_to_shared(c) + a * 4u));
    return v;
}
__device__ __forceinline__ uint4 ldr(const uint4* ring, uint32_t i) {
    uint4 v;
    asm volatile("ld.volatile.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "r"((uint32_t)__cvta_generic_to_shared(ring + (i & 2047u))));
    return v;
}
__device__ __forceinline__ int pick(int c0, int c1, int c2) { const bool L10 = c1 < c0; return (L10 ? c2 < c1 : c2 < c0) ? 2 : (L10 ? 1 : 0); }
__device__ __forceinline__ uint32_t sel(uint4 r, int k) { return k == 2 ? r.z : (k == 1 ? r.y : r.x); }

template <bool PAIR>
__global__ void chain(int* out, uint4* gout, int iters) {
    __shared__ int ctr[4096];
    __shared__ uint4 ring[2048];
    const uint32_t nt = blockDim.x, tid = threadIdx.x;
    for (int i = tid; i < 4096; i += nt) ctr[i] = i & 7;
    for (int i = tid; i < 2048; i += nt) {   // records: 3 brokers, and holders in the low bits of w (position in the topic)
        const uint32_t s = i * 2654435761u;
        ring[i] = make_uint4((s >> 3) & 4095, (s >> 9) & 4095, (s >> 15) & 4095, (s >> 21) % nt);
    }
    __syncthreads();
    int acc = 0;
    uint32_t base = 0;
    uint4 rp = ldr(ring, tid), rq = ldr(ring, nt + tid);
    uint4 h0 = ldr(ring, rq.w), h1 = ldr(ring, (rq.w + 1) % nt), h2 = ldr(ring, (rq.w + 2) % nt);
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
        if (!PAIR) {
            const int x0 = ld(ctr, rp.x), x1 = ld(ctr, rp.y), x2 = ld(ctr, rp.z);
            base += nt;
            const uint4 rn = ldr(ring, base + tid);
            const int k = pick(x0, x1, x2);
            const uint32_t oA = sel(rp, k);
            asm volatile("st.volatile.shared.s32 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(ctr) + oA * 4u),
                         "r"((k == 2 ? x2 : (k == 1 ? x1 : x0)) + 1) : "memory");
            gout[(size_t)(it & 1023) * nt + tid] = make_uint4(oA, rp.x, rp.y, rp.w);
            acc += oA;
            rp = rn;
            __syncthreads();
        } else {
            const int x0 = ld(ctr, rp.x), x1 = ld(ctr, rp.y), x2 = ld(ctr, rp.z);
            const int y0 = ld(ctr, rq.x), y1 = ld(ctr, rq.y), y2 = ld(ctr, rq.z);
            const uint32_t w0 = sel(h0, pick(ld(ctr, h0.x), ld(ctr, h0.y), ld(ctr, h0.z)));
            const uint32_t w1 = sel(h1, pick(ld(ctr, h1.x), ld(ctr, h1.y), ld(ctr, h1.z)));
            const uint32_t w2 = sel(h2, pick(ld(ctr, h2.x), ld(ctr, h2.y), ld(ctr, h2.z)));
            const uint32_t oA = sel(rp, pick(x0, x1, x2));
            const uint32_t oB = sel(rq, pick(y0 + (w0 == rq.x), y1 + (w1 == rq.y), y2 + (w2 == rq.z)));
            __syncthreads();
            asm volatile("red.shared.add.s32 [%0], 1;" ::"r"((uint32_t)__cvta_generic_to_shared(ctr) + oA * 4u) : "memory");
            asm volatile("red.shared.add.s32 [%0], 1;" ::"r"((uint32_t)__cvta_generic_to_shared(ctr) + oB * 4u) : "memory");
            gout[(size_t)(it & 511) * 2 * nt + tid] = make_uint4(oA, rp.x, rp.y, rp.w);
            gout[(size_t)(it & 511) * 2 * nt + nt + tid] = make_uint4(oB, rq.x, rq.y, rq.w);
            acc += oA + oB;
            base += 2 * nt;
            rp = ldr(ring, base + tid);
            rq = ldr(ring, base + nt + tid);
            h0 = ldr(ring, base + rq.w); h1 = ldr(ring, base + (rq.w + 1) % nt); h2 = ldr(ring, base + (rq.w + 2) % nt);
            __syncthreads();
        }
    }
    const long long t1 = clock64();
    if (tid == 0) { out[0] = acc; out[1] = (int)((t1 - t0) / iters); }
}

int main() {
    int* d; uint4* g;
    cudaMalloc(&d, 64); cudaMalloc(&g, (size_t)1024 * 256 * 16);
    const int iters = 20000;
    int h[2];
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    printf("%s\n", prop.name);
    for (int nt : {128, 256}) {
        chain<false><<<1, nt>>>(d, g, iters); cudaMemcpy(h, d, 8, cudaMemcpyDeviceToHost);
        const int lvl = h[1];
        chain<true><<<1, nt>>>(d, g, iters); cudaMemcpy(h, d, 8, cudaMemcpyDeviceToHost);
        printf("nt=%3d  level %4d cycles  pair step %4d cycles (two topics)  pair / level = %.2f  (gate: < 1.50)\n", nt, lvl, h[1],
               (double)h[1] / lvl);
    }
    printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
