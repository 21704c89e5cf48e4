// kassign_common.cuh — shared definitions of the sm_90a kernels of the kafka-assigner hot path.
//
// Reference being replaced (SURVEY.md §8a; KAS = KafkaAssignmentStrategy.java, KTA = KafkaTopicAssigner.java):
//   kassign_stage.cuh  ka_sticky_spread_kernel  KTA:49-69 (RF inference/validation), KAS:65-71 (capacity), KAS:73-99
//                                               (node/rack table), KAS:101-131 (sticky fill), KAS:133-160 (orphans),
//                                               KAS:162-200 (rotated first-fit spread), KAS:205-214 (ascending lists)
//                                               + the conflict levels the leader-order kernel is scheduled by
//   kassign_order.cuh  ka_order_levels_kernel   KAS:202-239 + PreferenceListOrderTracker KAS:244-302 against the
//                                               cross-topic Context.counter (KAS:360-369, KTA:19-23)
//                      ka_emit3_kernel          list positions -> ordered broker ids (KAS:229-235 output lists)
//
// Everything is integer indexing: no tensor cores. Tables and record streams are staged into shared memory with TMA
// bulk copies (cp.async.bulk + mbarrier); decisions that depend on the reference's visit order are taken with warp
// ballots / match / shuffles or under a barrier-separated schedule — never by an atomics race.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define KA_MAX_SLOTS 8      // max replicas per partition row (out_stride) on the fast paths
#define KA_DEAD 0xFFFFu     // "broker not in the live set" marker in 16-bit index space
#define KA_FULL 0xFFFFFFFFu

// The stable LSD radix passes (the wave documents' row grouping, the broker usage's event sort): 8-bit digits.
#define KA_RADIX_BITS 8
#define KA_RADIX_DIGITS (1 << KA_RADIX_BITS)
#define KA_RADIX_MIN_TILE 2048   // items per CTA of a pass, at least (a multiple of the 256 threads)
#define KA_RADIX_MAX_TILES 1024  // CTAs of a pass, at most: the (digit, tile) table stays within 256 k entries
static_assert(KA_RADIX_DIGITS == 256, "one thread per digit value");

// Error codes (mirror include/kassign.h)
#define KA_E_RF_MISMATCH 1
#define KA_E_RF_NOT_POSITIVE 2
#define KA_E_RF_GT_BROKERS 3
#define KA_E_UNASSIGNABLE 4
#define KA_E_HASH_INDEX 5

enum { KA_LUT_SMEM = 0, KA_LUT_GLOBAL = 1, KA_LUT_BSEARCH = 2 };

// One broker table in HBM: what kernel A stages and every id -> index lookup reads.
struct KaBrokers {
    int N, lut_mode, lut_off, blob_bytes, min_id;
    uint32_t range;
    const uint16_t* blob;       // rack16[Npad] || lut16[range_pad] (lut16 only when lut_mode == SMEM), 16B aligned; blob_bytes long
    const uint16_t* glut;       // lut_mode == KA_LUT_GLOBAL: lut16[range]
    const int32_t* broker_id;   // [N] ascending
};

// What kernel A writes for a run (rows and topics relative to the run's block).
struct KaStageOut {
    unsigned char* rec;         // [Q] partition records in schedule order (16 B for rec_kind 3, else 32 B)
    uint16_t* perm;             // [Q] LEVELS && rec_kind == 3: partition ordinal (inside its topic) of each schedule position
    int32_t* ntl;               // [T] LEVELS: number of chunks of each topic
    uint32_t* lend;             // [Q] LEVELS: lend[g0 + i] = topic-relative end of the topic's i-th chunk (first ntl[t] entries)
    int4* tstatus;              // [T] per-topic error record (written only on error)
    unsigned* err_topic;        // unsigned atomicMin of the failing topic index (init = 0xFFFFFFFF)
};

// One member of a batched solve, in HBM: its broker table, its own fresh Context, its window of the call's shared input and
// its slice of the call's scratch. A member is a candidate broker table over the whole input (ka_solve_candidates: t0 = 0,
// T = the call's topics, row0 = 0, records from k * Q) or one cluster of a fleet (ka_solve_clusters: its own topics and rows,
// records at their input rows). Every kernel of the batched solve reads the entry of its member once, at entry; the kernels of
// the single solve never see one.
struct KaCandidate {
    KaBrokers br;
    KaStageOut out;             // rec / perm / lend indexed by input row, ntl / tstatus / err_topic by input topic
    int32_t* ctr8;              // [N+1][8] the member's Context.counter (+ the chains' dummy row), zero at the call's start
    const int32_t* loff;        // [T+1] LEVELS: first chunk of each of the member's topics in the call-wide chunk table
    uint32_t pos0;              // LEVELS: position of the member's first record in the call-wide chunk table
    int t0, T;                  // the member's topics: [t0, t0 + T) of the shared input
    uint32_t row0, Q;           // the member's rows: [row0, row0 + Q) of the shared input (part_off[t0] ..)
    int desired_rf;             // the member's --desired_replication_factor (-1: keep)
};

// Broker id -> index in the ascending table br (KA_DEAD when absent). lut: br's SMEM-mode LUT, wherever it is read from.
__device__ __forceinline__ uint32_t ka_lookup(int id, const uint16_t* lut, const KaBrokers& br) {
    if (br.lut_mode == KA_LUT_SMEM) {
        uint32_t off = (uint32_t)id - (uint32_t)br.min_id;
        return off < br.range ? (uint32_t)lut[off] : KA_DEAD;
    } else if (br.lut_mode == KA_LUT_GLOBAL) {
        uint32_t off = (uint32_t)id - (uint32_t)br.min_id;
        return off < br.range ? (uint32_t)__ldg(&br.glut[off]) : KA_DEAD;
    } else {
        int lo = 0, hi = br.N - 1;
        while (lo <= hi) {
            int mid = (lo + hi) >> 1;
            int v = __ldg(&br.broker_id[mid]);
            if (v == id) return (uint32_t)mid;
            if (v < id) lo = mid + 1; else hi = mid - 1;
        }
        return KA_DEAD;
    }
}

// ------------------------------------------------------------------------------------------------
// Partition records: what kernel A hands to the leader-order kernel, in SCHEDULE order (topic by topic; inside a
// topic by conflict level, then partition ascending). Broker indices are positions in the ascending live-id table.
//   rows of <= 3 replicas  uint4 {a0, a1, a2, f}: a_j = (index of the broker at position j of the slot-0 scan order of
//                          KAS:267, i.e. ascending list position i sits at j = (i + |hash| % len) % len) << 2 = byte offset
//                          of that broker's counter in a 4-byte column; unused slots = the dummy broker N;
//                          f = len[0:2) | e01[2] | e02[3] | e12[4] | first-of-level[7], e_pq = tie-break of the slot-1 scan over the pair
//                          (p, q) left when the third position took slot 0 (see kassign_stage.cuh / kassign_order.cuh).
//                          The slot-0 chain rewrites it as {op, oq, len | e << 2, o0} (remaining pair in scan order, its
//                          tie-break, the slot-0 broker); the slot-1 chain as the ordered list {o0, o1, o2, len | e << 2}.
//   rows of 4..8           2 x uint4 : {idx0|idx1<<16, idx2|idx3<<16, idx4|idx5<<16, idx6|idx7<<16}, {meta32, row, 0, 0}
//                          meta32 = len[0:4) | rotations for k = 2..8 (ka_rot_bits), row = block-relative output row
// ------------------------------------------------------------------------------------------------


// ------------------------------------------------------------------------------------------------
// small PTX helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ka_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void ka_mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(ka_smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void ka_fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void ka_fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void ka_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(ka_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void ka_mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(ka_smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// TMA bulk copy global -> shared (non-tensor form). bytes % 16 == 0, both addresses 16B aligned.
__device__ __forceinline__ void ka_tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     ka_smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(ka_smem_u32(bar))
                 : "memory");
}

__device__ __forceinline__ int4 ka_ldg_stream_v4(const int4* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

__device__ __forceinline__ uint32_t ka_lanemask_lt() {
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

// The sum of v over the lanes of `grp` (this lane among them), in every lane of the group. Needs v >= 0 in every lane and a
// sum <= INT64_MAX. v goes in three limbs of at most 22 bits, so a 32-bit __reduce_add_sync over at most 32 lanes never
// carries; any group of lanes, the whole warp included.
__device__ __forceinline__ long long ka_group_sum64(long long v, unsigned grp) {
    const unsigned long long u = (unsigned long long)v;
    const unsigned long long a0 = __reduce_add_sync(grp, (unsigned)(u & 0x3FFFFFu));
    const unsigned long long a1 = __reduce_add_sync(grp, (unsigned)(u >> 22 & 0x1FFFFFu));
    const unsigned long long a2 = __reduce_add_sync(grp, (unsigned)(u >> 43));
    return (long long)(a0 + (a1 << 22) + (a2 << 43));
}

// Exclusive scan of in[0..n) by ONE CTA of 1024 threads, in rounds of 1024 elements: out[i] = carry + in[0] + .. + in[i - 1]
// (in T, then narrowed to Out). Returns carry + the sum of all n, in every thread. in and out may be the same array.
template <typename T, typename In, typename Out>
__device__ __forceinline__ T ka_cta_scan(const In* in, Out* out, int n, T carry) {
    __shared__ T wtot[32];
    __shared__ T run;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) run = carry;
    __syncthreads();
    for (int b0 = 0; b0 < n; b0 += 1024) {
        const int b = b0 + threadIdx.x;
        const T v = b < n ? (T)in[b] : (T)0;
        T x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const T y = __shfl_up_sync(KA_FULL, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) wtot[warp] = x;
        __syncthreads();
        if (warp == 0) {
            T w = wtot[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const T y = __shfl_up_sync(KA_FULL, w, o);
                if (lane >= o) w += y;
            }
            wtot[lane] = w;  // inclusive over warps
        }
        __syncthreads();
        const T base = run + (warp > 0 ? wtot[warp - 1] : (T)0);
        if (b < n) out[b] = (Out)(base + x - v);
        __syncthreads();
        if (threadIdx.x == 1023) run = base + x;
        __syncthreads();
    }
    return run;
}

// Rotation bits of one topic: (|hash| % k) for k = 2..8 packed above the 4-bit length (KAS:190 applied
// to the remaining-set sizes of KAS:267). Layout: len[0:4) k2[4] k3[5:7) k4[7:9) k5[9:12) k6[12:15) k7[15:18) k8[18:21)
__device__ __forceinline__ uint32_t ka_rot_bits(uint32_t habs) {
    return ((habs % 2u) << 4) | ((habs % 3u) << 5) | ((habs % 4u) << 7) | ((habs % 5u) << 9) | ((habs % 6u) << 12) |
           ((habs % 7u) << 15) | ((habs % 8u) << 18);
}
template <int RS>
__device__ __forceinline__ int ka_rot_of(uint32_t meta, int k) {
    // k in [1,RS]; select chain instead of a table so nothing lands in local memory
    int s = 0;
    if (k == 2) s = (meta >> 4) & 1u;
    if (k == 3) s = (meta >> 5) & 3u;
    if (k == 4) s = (meta >> 7) & 3u;
    if (RS > 4) {
        if (k == 5) s = (meta >> 9) & 7u;
        if (k == 6) s = (meta >> 12) & 7u;
        if (k == 7) s = (meta >> 15) & 7u;
        if (k == 8) s = (meta >> 18) & 7u;
    }
    return s;
}
