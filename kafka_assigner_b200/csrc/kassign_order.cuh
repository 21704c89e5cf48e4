// kassign_order.cuh — leader-preference ordering (KAS:202-239, PreferenceListOrderTracker KAS:244-302) against the
// cross-topic Context.counter (KAS:360-369, KTA:19-23), as a LEVEL-SYNCHRONOUS schedule.
//
// Context.counter is shared by every topic of a run (KAG:172), so leader ordering is one serial chain over all partitions
// of all topics; two partitions commute iff their broker sets are disjoint. Kernel A sorted every topic's partitions into
// conflict levels (kassign_stage.cuh): the partitions of one level touch pairwise disjoint counter rows. This kernel
// walks the levels in order with ONE CTA: a level is processed by all threads in parallel (read the three counter rows,
// take the KAS:226-234 decision, bump counter[list[r]][r]), levels are separated by one `bar.sync 0` (or __syncwarp when
// the CTA is a single warp). No tickets, no polling: cost per level = LDS + decision + STS + barrier.
// The partition records arrive through a TMA ring (cp.async.bulk into shared memory, one mbarrier per stage, refilled by
// thread 0 once per stage), so global latency never touches the chain.
#pragma once
#include "kassign_common.cuh"

// ------------------------------------------------------------------------------------------------
// Chunk tables (only when some topic has more than one level; otherwise level L = topic L = records [L*P, (L+1)*P)).
// A chunk = at most W consecutive records of ONE level (W = consumer threads of the order kernel).
//   ntl[t]  chunks of topic t            -> loff[t] = exclusive scan (loff[T] = number of chunks of the block)
//   lend[g0 + i] topic-relative ends     -> chunk_end[loff[t] + i] = g0 + lend[g0 + i]   (block-relative record positions)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) ka_level_scan_kernel(const int32_t* __restrict__ ntl, int T, int32_t* __restrict__ loff) {
    const int total = ka_cta_scan(ntl, loff, T, 0);
    if (threadIdx.x == 0) loff[T] = total;
}

// Chunk ends of a chunk table of U topics, one warp per topic. Topic u = k * T + t (k > 0 only in a batched solve over
// candidates: the K candidates' tables are one table of K * T topics) starts at record k * rows + part_off[t] (dense: t * P),
// rows = the records of one candidate. The clusters of a fleet are one table of their U = T topics (rows = 0): topic u's
// records start at part_off[u].
__global__ void __launch_bounds__(256) ka_level_fill_kernel(const int32_t* __restrict__ ntl, const int32_t* __restrict__ loff,
                                                            const uint32_t* __restrict__ lend, const int64_t* __restrict__ part_off, int P,
                                                            int T, int U, int64_t rows, uint32_t* __restrict__ lvl_end) {
    const int lane = threadIdx.x & 31;
    const int u = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (u >= U) return;
    const int k = u / T, t = u - k * T;
    const int64_t g0 = (int64_t)k * rows + (part_off ? part_off[t] : (int64_t)t * P);
    const int d = ntl[u], o = loff[u];
    for (int l = lane; l < d; l += 32) lvl_end[o + l] = (uint32_t)g0 + lend[g0 + l];
}

// ------------------------------------------------------------------------------------------------
struct KaOrderParams {
    uint32_t Q;                 // records (partitions) of the block
    int N;
    int S;                      // output row stride (generic kinds write rows themselves)
    const void* rec;            // schedule-order records (16 B for rows <= 3, else 32 B), 16B aligned. Rows <= 3: each
                                // record is overwritten in place: {p, q, len|e, leader} by the slot-0 chain, the ordered list
                                // {o0, o1, o2, f} (o_r = broker index << 2) by the slot-1 chain
    uint32_t uniform_width;     // > 0: level L = records [L*w, (L+1)*w), cut into chunks of blockDim records;  0: chunk table
    const uint32_t* chunk_end;  // table mode: end position of each chunk of the STAGED block (a chunk never spans two levels)
    const int32_t* chunk_lo_ptr;  // device scalars: this launch walks chunks [*chunk_lo_ptr, *chunk_hi_ptr) of that table
    const int32_t* chunk_hi_ptr;  //   (loff[] of ka_level_scan_kernel at the first / one-past-last topic of the launch)
    uint32_t pos_base;          // record position of p.rec[0] inside the staged block (chunk_end values are block-relative)
    int32_t* ctr8;              // [N][8] Context.counter for the current broker table (in/out)
    const int32_t* broker_id;   // RS > 3: rows are written by this kernel
    int32_t* out;
    int32_t* out_len;
    int ring_log2;              // log2(records per ring stage)
    // batched solve (CAND): CTA k orders batch member k. N / ctr8 / records / chunk table come from cand[k]: the launch walks
    // the member's records [pos_base, pos_base + Q) and chunks [loff[cand_t0], loff[cand_t1]) of its chunk table, both
    // clipped to the member's window (its cand[k].Q records, cand[k].T topics).
    const KaCandidate* cand;
    int cand_t0, cand_t1;
};

#define KA_RING_STAGES 8

__device__ __forceinline__ void ka_mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(ka_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void ka_named_bar_sync(uint32_t id, uint32_t nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// Programmatic dependent launch: wait until the grid this one was launched behind has completed and its writes are visible
// (returns at once without such a predecessor); let the grid launched behind this one start its prologue.
__device__ __forceinline__ void ka_grid_dependency_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void ka_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// counter-row access: shared memory (byte address = base + idx*16 .. the record's precomputed offset) or global memory
// (ctr8 rows of 8 ints, L2-resident; for broker tables beyond shared memory)
template <bool GCTR> struct KaCtr;
template <> struct KaCtr<false> {
    typedef uint32_t H;
    // a = idx << 4 (record field); CW ints per row in shared memory
    template <int CW> static __device__ __forceinline__ H row(uint32_t sbase, int32_t*, uint32_t a) { return sbase + (CW == 4 ? a : a * 2u); }
    static __device__ __forceinline__ int4 ld4(H h, int off) {
        int4 v;
        asm volatile("ld.volatile.shared.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(h + off));
        return v;
    }
    static __device__ __forceinline__ void st(H h, int off, int v) { asm volatile("st.volatile.shared.s32 [%0], %1;" ::"r"(h + off), "r"(v) : "memory"); }
    // slot chains: one counter column in shared memory, a = idx << 2
    static __device__ __forceinline__ H col(uint32_t sbase, int32_t*, uint32_t a, int) { return sbase + a; }
    static __device__ __forceinline__ int ld1(H h) {
        int v;
        asm volatile("ld.volatile.shared.s32 %0, [%1];" : "=r"(v) : "r"(h));
        return v;
    }
    static __device__ __forceinline__ void st1(H h, int v) { asm volatile("st.volatile.shared.s32 [%0], %1;" ::"r"(h), "r"(v) : "memory"); }
};
template <> struct KaCtr<true> {
    typedef char* H;
    template <int CW> static __device__ __forceinline__ H row(uint32_t, int32_t* g, uint32_t a) { return reinterpret_cast<char*>(g) + (size_t)a * 2u; }
    static __device__ __forceinline__ int4 ld4(H h, int off) {
        int4 v;
        asm volatile("ld.volatile.global.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(h + off));
        return v;
    }
    static __device__ __forceinline__ void st(H h, int off, int v) { asm volatile("st.volatile.global.s32 [%0], %1;" ::"l"(h + off), "r"(v) : "memory"); }
    static __device__ __forceinline__ H col(uint32_t, int32_t* g, uint32_t a, int slot) { return reinterpret_cast<char*>(g) + (size_t)a * 8u + slot * 4; }
    static __device__ __forceinline__ int ld1(H h) {
        int v;
        asm volatile("ld.volatile.global.s32 %0, [%1];" : "=r"(v) : "l"(h));
        return v;
    }
    static __device__ __forceinline__ void st1(H h, int v) { asm volatile("st.volatile.global.s32 [%0], %1;" ::"l"(h), "r"(v) : "memory"); }
};

// One selection pass of KAS:263-278 for rows of up to RS replicas (array form; rows of <= 3 use the scalar code below).
template <int RS>
__device__ __forceinline__ void ka_order_generic(const int (&c)[RS][RS], int len, uint32_t meta, int (&perm)[RS]) {
    uint32_t remmask = (1u << len) - 1u;
#pragma unroll
    for (int r = 0; r < RS; ++r) {
        if (r < len) {
            const int k = len - r;
            const int s = ka_rot_of<RS>(meta, k);
            long long best = 0x7FFFFFFFFFFFFFFFLL;
            int bpos = 0;
#pragma unroll
            for (int pos = 0; pos < RS; ++pos) {
                if ((remmask >> pos) & 1u) {
                    int j = __popc(remmask & ((1u << pos) - 1u)) + s;  // position in the rotated scan (KAS:267)
                    if (j >= k) j -= k;
                    const long long key = (long long)c[pos][r] * 8 + j;  // strict <, ties to the earlier scan position
                    if (key < best) { best = key; bpos = pos; }
                }
            }
            perm[r] = bpos;
            remmask &= ~(1u << bpos);
        }
    }
}

// KIND 0 / 1 = slot-0 / slot-1 chain of rows <= 3 (16-byte records, rewritten in place), 4 = rows of 4, 8 = rows of 5..8
// (32-byte records, all slots in one chain, rows written directly). blockDim = NT threads.
//   record ring     thread 0 streams the records into a ring of KA_RING_STAGES shared-memory stages with cp.async.bulk (TMA);
//                   full[stage] mbarriers carry the byte count; a stage is refilled as soon as the level barrier shows that
//                   every thread is done with it
//   all threads     chunk by chunk (<= NT records, never spanning two levels): thread i takes record i of the chunk,
//                   loads its counter rows, decides, stores the bumps; ONE `bar.sync 0` per chunk is the only
//                   synchronisation on the chain. The next chunk's record is read from the ring before the barrier.
//   CAND            (slot chains only) a batched solve: CTA k orders candidate k, whose values (p.cand[k]) are read once at
//                   entry; rec / ctr8 then take the same round trip into registers as the other invariants
template <int KIND, bool GCTR, int MAXNT, bool SINGLE, bool WARP1, bool FULL, bool CAND = false>
__global__ void __launch_bounds__(MAXNT, 1) ka_order_levels_kernel(const KaOrderParams p) {
    constexpr int RS = KIND <= 1 ? 3 : KIND;                 // KIND 0 / 1: slot-0 / slot-1 chain of rows <= 3; 4 / 8: rows of 4 / 5..8
    constexpr int CW = KIND <= 1 ? 1 : (KIND == 4 ? 4 : 8);  // ints per broker in shared memory (one counter column for the slot chains)
    constexpr int RB = RS == 3 ? 16 : 32;                    // record bytes
    constexpr int NS = KA_RING_STAGES;
    typedef KaCtr<GCTR> C;
    extern __shared__ __align__(128) unsigned char ka_osmem[];
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    unsigned char* ring = ka_osmem;
    uint64_t* full = reinterpret_cast<uint64_t*>(ka_osmem + ((size_t)NS << p.ring_log2) * RB);
    volatile uint32_t* pin = reinterpret_cast<volatile uint32_t*>(full + 2 * NS);   // 16 words
    int* ctr = reinterpret_cast<int*>(ka_osmem + ((size_t)NS << p.ring_log2) * RB + 256);
    static_assert(!CAND || KIND <= 1, "batched solves order rows of <= 3 replicas");
    const KaCandidate* const cd = CAND ? p.cand + blockIdx.x : nullptr;
    // no broker: every topic of the member failed in kernel A; no record of the member in the launch's window: nothing to order
    if (CAND && (cd->br.N <= 0 || p.pos_base >= cd->Q)) return;
    // Loop invariants take a round trip through shared memory (volatile) so that they live in registers: ptxas otherwise
    // re-reads kernel parameters from the constant bank inside the chain loop, and every such load stalls a branch.
    if (tid == 0) {
        const void* const rec = CAND ? (const void*)(cd->out.rec + ((size_t)cd->row0 + p.pos_base) * RB) : p.rec;
        int32_t* const c8 = CAND ? cd->ctr8 : p.ctr8;
        pin[0] = CAND ? min(p.Q, cd->Q - p.pos_base) : p.Q;   // CAND: the launch's window clipped to the member's rows
        pin[1] = blockDim.x; pin[2] = (uint32_t)p.ring_log2; pin[3] = p.uniform_width;
        pin[4] = (uint32_t)reinterpret_cast<uintptr_t>(rec); pin[5] = (uint32_t)(reinterpret_cast<uintptr_t>(rec) >> 32);
        pin[6] = (uint32_t)reinterpret_cast<uintptr_t>(c8); pin[7] = (uint32_t)(reinterpret_cast<uintptr_t>(c8) >> 32);
        if (CAND) pin[8] = (uint32_t)cd->br.N;
    }
    __syncthreads();
    const uint32_t Q = pin[0], NT = pin[1];
    const int LG = (int)pin[2];
    const uint32_t w = pin[3];
    uint4* const orec = reinterpret_cast<uint4*>((uintptr_t)pin[4] | ((uintptr_t)pin[5] << 32));
    int32_t* const ctr8 = reinterpret_cast<int32_t*>((uintptr_t)pin[6] | ((uintptr_t)pin[7] << 32));
    const uint32_t G = 1u << LG;

    if (tid == 0) {
        for (int i = 0; i < NS; ++i) ka_mbar_init(&full[i], 1);
        ka_fence_mbar_init();
    }
    // idle lanes read (and ignore) ring slots past the end of the stream: make those valid records (all zero). Every lane of
    // the FULL shape is active on every chunk, and its one read past the end (the last chunk's prefetch) is never used.
    if (!FULL)
        for (uint32_t i = tid; i < (uint32_t)NS * G * (RB / 16); i += blockDim.x) reinterpret_cast<uint4*>(ring)[i] = make_uint4(0, 0, 0, 0);
    ka_fence_proxy_async();   // generic-proxy writes above vs the async-proxy (TMA) writes that follow
    __syncthreads();

    // ---- record ring: stage j of the stream lives in slot j % NS. Thread 0 issues the TMA copies: the first NS stages here,
    //      stage j + NS as soon as every thread is done with stage j (the "hand-over", once per stage, off the per-level path).
    //      No producer warp and no empty-barriers: the level barrier already tells thread 0 that a stage is consumed, and with
    //      every thread of the CTA a consumer the level barrier is the plain `bar.sync 0` (measurably cheaper than a named
    //      barrier with a register thread count — tests/tools/micro/level_floor.cu).
    const uint32_t nstages_all = (Q + G - 1) >> LG;
    auto issue_stage = [&](uint32_t j) {   // thread 0 only
        const uint32_t slot = j & (NS - 1);
        const uint32_t bytes = min(G, Q - (j << LG)) * RB;
        ka_mbar_expect_tx(&full[slot], bytes);
        ka_tma_bulk_g2s(ring + (size_t)slot * G * RB, reinterpret_cast<const unsigned char*>(CAND ? (const void*)orec : p.rec) + (size_t)j * G * RB,
                        bytes, &full[slot]);
    };
    if (tid == 0)
        for (uint32_t j = 0; j < min(nstages_all, (uint32_t)NS); ++j) issue_stage(j);

    // Everything above reads only parameters and records, which kernel A or the slot-0 chain wrote and the stream has joined
    // through events. The counters are the output of the chain launch before this one on the stream, which may still be
    // running when this grid was launched behind it (programmatic dependent launch): only their load waits for it.
    ka_grid_dependency_wait();
    if (!GCTR)
        for (uint32_t i = tid; i < (uint32_t)(CAND ? (int)pin[8] : p.N) * CW; i += blockDim.x)
            ctr[i] = ctr8[(i / CW) * KA_MAX_SLOTS + (KIND <= 1 ? KIND : (int)(i % CW))];
    if (KIND <= 1 && tid == 0) {  // the dummy broker (index N) that pads rows shorter than 3: a counter that never wins a comparison
        // INT_MAX, and every record lists the dummy after its real brokers: a real counter is at most INT_MAX, so it wins both
        // the slot-0 minimum and the slot-1 pair (e = 0 there) in scan order. The dummy is never bumped (the bumps below are
        // skipped for rows too short to fill the slot), so its counter stays INT_MAX for the whole launch.
        const int N = CAND ? (int)pin[8] : p.N;
        if (GCTR) ctr8[(size_t)N * KA_MAX_SLOTS + KIND] = 0x7FFFFFFF; else ctr[N] = 0x7FFFFFFF;
    }
    __syncthreads();

    // ---- consumers ------------------------------------------------------------------------------------------------------
    const uint32_t rmask = (uint32_t)NS * G - 1u;
    const uint32_t ring_s = ka_smem_u32(ring);
    uint32_t landed = 0;    // stages this thread has seen complete
    uint32_t released = 0;  // thread 0: stages handed back to the producer
    // chunk boundaries
    const int chunk_lo = w ? 0 : (CAND ? cd->loff[min(p.cand_t0, cd->T)] : *p.chunk_lo_ptr);
    const int nchunk = w ? 0 : (CAND ? cd->loff[min(p.cand_t1, cd->T)] : *p.chunk_hi_ptr) - chunk_lo;
    const uint32_t* const cend = p.chunk_end + chunk_lo;
    const uint32_t pos_base = CAND ? cd->pos0 + p.pos_base : p.pos_base;
    int wbase = 0;
    uint32_t wcur = Q, wnxt = Q;  // table mode: chunk end of chunk wbase + lane, wbase + 32 + lane
    if (!w) {
        wcur = (int)lane < nchunk ? cend[lane] - pos_base : Q;
        wnxt = 32 + (int)lane < nchunk ? cend[32 + lane] - pos_base : Q;
    }
    uint32_t lvl_hi = w;  // uniform mode: end of the level the current chunk belongs to
    int c = 0;            // chunk ordinal (table mode)
    auto next_end = [&](uint32_t cur_end) -> uint32_t {  // end of the chunk that starts at cur_end (warp-uniform)
        if (w) {
            if (cur_end == lvl_hi) lvl_hi += w;
            return min(min(cur_end + NT, lvl_hi), Q);
        }
        ++c;
        if (c >= nchunk) return Q;
        if (c >= wbase + 32) {
            wcur = wnxt;
            wbase += 32;
            const int i = wbase + 32 + (int)lane;
            wnxt = i < nchunk ? cend[i] - pos_base : Q;
        }
        return __shfl_sync(KA_FULL, wcur, c - wbase);
    };
    auto read_rec = [&](uint32_t pos, uint4& a, uint4& b) {
        const uint32_t src = ring_s + (pos & rmask) * RB;
        asm volatile("ld.volatile.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w) : "r"(src));
        if (RS != 3) asm volatile("ld.volatile.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w) : "r"(src + 16));
    };
    auto cross = [&](uint32_t held_end, uint32_t xlast) {
        // entering a new ring stage: hand finished stages back FIRST (every record below held_end is already in registers or
        // done), then wait for the stage(s) the next chunk needs
        if (tid == 0 && ((released + 1u) << LG) <= held_end) {
            ka_fence_proxy_async();   // generic-proxy reads of the slot (all complete: a level barrier separates them) vs the TMA write
            while (((released + 1u) << LG) <= held_end) {
                if (released + NS < nstages_all) issue_stage(released + NS);
                ++released;
            }
        }
        const uint32_t j = xlast >> LG;
        while (landed <= j) { ka_mbar_wait(&full[landed & (NS - 1)], (landed / NS) & 1u); ++landed; }
    };

    const uint32_t cbase = GCTR ? 0u : ka_smem_u32(ctr);
    uint32_t start = 0, end = w ? min(min(NT, w), Q) : (nchunk > 0 ? __shfl_sync(KA_FULL, wcur, 0) : Q);
    uint32_t limit = 0;   // first record position whose ring stage this thread has not seen land yet
    auto cross_to = [&](uint32_t held_end, uint32_t nend) {
        cross(held_end, nend - 1u);
        limit = landed << LG;
    };
    uint4 ra0 = make_uint4(0, 0, 0, 0), ra1 = ra0, rb0 = ra0, rb1 = ra0;
    cross_to(0, end);
    read_rec(start + tid, ra0, ra1);

    // ---- slot chains (rows <= 3) ------------------------------------------------------------------------------------------
    // slot-0 chain: record = {a0, a1, a2, f}: a_j = (index of the broker at position j of the rotated scan of KAS:267) << 2 =
    //   byte offset of its counter in a column; rows shorter than 3 are padded with the DUMMY broker (index N, "infinite"
    //   counter: always ordered last, so no length dispatch); f = len[0:2) | e01[2] | e02[3] | e12[4]. Slot 0 reads and bumps
    //   ONLY counter[.][0] (getLeastSeenNodeForReplicaId(0, .), KAS:263-278), so this chain does not wait for the slot-1
    //   decisions: it hands {remaining pair, tie-break, leader} to the slot-1 chain in place of the record.
    // slot-1 chain: record = {op, oq, f, oA}: the two brokers left after slot 0 in scan order, f = len[0:2) | e[2], the slot-0
    //   broker. q takes slot 1 iff c_q < c_p + e (e folds the ascending-id order and |hash| % 2 of the second
    //   getNodeProcessingOrder call, KAS:267); only counter[.][1] is read and bumped. The last broker's counter[.][2] is
    //   write-only for rows <= 3: ka_emit3_kernel adds it in parallel.
    // Idle lanes compute on a stale (valid) record and store nothing.
#define KA_SLOT0_CORE(RC, ACTIVE, POS)                                                                                          \
            const uint32_t a0 = RC.x, a1 = RC.y, a2 = RC.z, f = RC.w;                                                           \
            const int x0 = C::ld1(C::col(cbase, ctr8, a0, 0)), x1 = C::ld1(C::col(cbase, ctr8, a1, 0)), x2 = C::ld1(C::col(cbase, ctr8, a2, 0));
#define KA_SLOT0_DECIDE(ACTIVE, POS)                                                                                            \
            /* strict minimum in scan order, ties to the earlier scan position: the record IS in scan order. Written as a   \
               min tree (x2 wins iff it is below the winner of x0 / x1): the bump's address and value are three dependent   \
               steps behind the loads, the rewritten record six; the level barrier waits for both (DESIGN §2 B) */          \
            const bool L10 = x1 < x0;                                                                                       \
            const int m01 = min(x0, x1);                                                                                    \
            const bool is2 = x2 < m01;                                                                                      \
            const uint32_t oA = is2 ? a2 : (L10 ? a1 : a0);                                                                 \
            const int vA = min(m01, x2);                                                                                    \
            /* remaining pair (p, q), p < q in scan order, and f with the tie-break e_pq of its slot-1 scan at bit 2        \
               (e01 / e02 / e12 at bits 2 / 3 / 4 when 2 / 1 / 0 wins) */                                                   \
            const uint32_t op = is2 ? a0 : (L10 ? a0 : a1), oq = is2 ? a1 : a2;                                             \
            const uint32_t fz = f & 0x83u;                                                                                  \
            const uint32_t fo = is2 ? (fz | (f & 4u)) : (L10 ? (fz | ((f >> 1) & 4u)) : (fz | ((f >> 2) & 4u)));            \
            if (ACTIVE) {                                                                                                       \
                if (f & 3u) C::st1(C::col(cbase, ctr8, oA, 0), vA + 1);   /* counter[list[0]][0] += 1 (KAS:254-261); never the dummy */ \
                asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(orec + (POS)), "r"(op), "r"(oq), "r"(fo), "r"(oA) : "memory"); \
            }
#define KA_SLOT1_CORE(RC, ACTIVE, POS)                                                                                          \
            const uint32_t op = RC.x, oq = RC.y, f = RC.z, oA = RC.w;                                                           \
            const int yp = C::ld1(C::col(cbase, ctr8, op, 1)), yq = C::ld1(C::col(cbase, ctr8, oq, 1));
#define KA_SLOT1_DECIDE(ACTIVE, POS)                                                                                            \
            const bool pickq = yq < yp + (int)((f >> 2) & 1u);                                                                  \
            const uint32_t o1 = pickq ? oq : op, o2 = pickq ? op : oq;                                                          \
            if (ACTIVE) {                                                                                                       \
                /* counter[list[1]][1] += 1 (KAS:254-261), for rows of >= 2: a shorter row's pair is the dummy twice */          \
                if (f & 2u) C::st1(C::col(cbase, ctr8, o1, 1), (pickq ? yq : yp) + 1);                                          \
                /* the ordered list replaces the record (ka_emit3_kernel reads it) */                                           \
                asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(orec + (POS)), "r"(oA), "r"(o1), "r"(o2), "r"(f) : "memory"); \
            }
    if (KIND <= 1 && WARP1) {
        // ---- single consumer warp (narrow levels): WINDOW mode. 32 consecutive records per iteration; bit 7 of f marks the
        //      first record of a level, so the window splits into level groups by one ballot — no chunk table. Only the
        //      counter-critical part (load, compare, bump) runs once per group, separated by __syncwarp; everything that does
        //      not touch the counters (remaining pair, tie-break, record store) runs once per window at full width. -----------
        const uint32_t lmle = ka_lanemask_lt() | (1u << lane);
        for (uint32_t wstart = 0; wstart < Q;) {
            const uint32_t pos = wstart + tid;
            const uint32_t f = KIND == 0 ? ra0.w : ra0.z;
            const uint32_t bal = __ballot_sync(KA_FULL, pos < Q && (f & 0x80u)) | 1u;   // lane 0 continues or opens a group
            // (cutting windows at level boundaries — whole levels only — was measured: fewer groups but more windows, slower)
            const int ngrp = __popc(bal);
            const uint32_t take = 32u;
            const bool active = pos < Q;
            const int grp = __popc(bal & lmle) - 1;
            const uint32_t nstart = wstart + take, need = min(nstart + 32u, Q);
            if (__builtin_expect(need > limit, 0)) cross_to(nstart, need);   // rare: the next window enters a new ring stage
            read_rec(nstart + tid, rb0, rb1);
            if (KIND == 0) {
                const uint32_t a0 = ra0.x, a1 = ra0.y, a2 = ra0.z;
                bool is1 = false, is2 = false;
                for (int g = 0; g < ngrp; ++g) {
                    if (grp == g && active) {
                        const int x0 = C::ld1(C::col(cbase, ctr8, a0, 0)), x1 = C::ld1(C::col(cbase, ctr8, a1, 0)), x2 = C::ld1(C::col(cbase, ctr8, a2, 0));
                        const bool L10 = x1 < x0, L20 = x2 < x0, L21 = x2 < x1;   // scan order: strict '<', ties to the earlier
                        is2 = L10 ? L21 : L20;
                        is1 = L10 && !L21;
                        if (f & 3u) C::st1(C::col(cbase, ctr8, is2 ? a2 : (is1 ? a1 : a0), 0), (is2 ? x2 : (is1 ? x1 : x0)) + 1);   // KAS:254-261
                    }
                    __syncwarp();   // level barrier
                }
                const bool is0 = !(is1 || is2);
                const uint32_t oA = is2 ? a2 : (is1 ? a1 : a0), op = is0 ? a1 : a0, oq = is2 ? a1 : a2;
                const uint32_t esh = is2 ? f : (is1 ? f >> 1 : f >> 2);
                if (active) asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(orec + pos), "r"(op), "r"(oq), "r"((f & 0x83u) | (esh & 4u)), "r"(oA) : "memory");
            } else {
                const uint32_t op = ra0.x, oq = ra0.y, oA = ra0.w;
                bool pickq = false;
                for (int g = 0; g < ngrp; ++g) {
                    if (grp == g && active) {
                        const int yp = C::ld1(C::col(cbase, ctr8, op, 1)), yq = C::ld1(C::col(cbase, ctr8, oq, 1));
                        pickq = yq < yp + (int)((f >> 2) & 1u);
                        if (f & 2u) C::st1(C::col(cbase, ctr8, pickq ? oq : op, 1), (pickq ? yq : yp) + 1);   // KAS:254-261
                    }
                    __syncwarp();
                }
                if (active) asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(orec + pos), "r"(oA), "r"(pickq ? oq : op), "r"(pickq ? op : oq), "r"(f) : "memory");
            }
            ra0 = rb0;
            wstart = nstart;
        }
    } else if (KIND <= 1 && SINGLE) {
        // ---- capacity 1 and P <= CTA: chunk k = topic k = records [k*w, (k+1)*w). The inner loop has NO bounds logic: the
        //      number of chunks that can run before the next ring-stage hand-over is computed outside it. ---------------------
        const uint32_t nchunks = Q / w, nstages = (Q + G - 1) >> LG;
        const uint32_t w16 = w * RB, rmask16 = (uint32_t)NS * G * RB - 1u;
        const bool act = FULL || tid < w;       // loop-invariant: every chunk is full (Q = T * w); FULL: w == NT, no idle lane at all
        uint32_t roff = (tid * RB) & rmask16;   // ring byte offset of my record of the current chunk
        uint32_t pos = tid, k = 0;
#define KA_SINGLE_BODY(RC, RN)                                                                                                  \
        {                                                                                                                       \
            if (KIND == 0) {                                                                                                    \
                KA_SLOT0_CORE(RC, act, pos)                                                                                     \
                roff = (roff + w16) & rmask16;                                                                                  \
                asm volatile("ld.volatile.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(RN.x), "=r"(RN.y), "=r"(RN.z), "=r"(RN.w) : "r"(ring_s + roff)); \
                KA_SLOT0_DECIDE(act, pos)                                                                                       \
            } else {                                                                                                            \
                KA_SLOT1_CORE(RC, act, pos)                                                                                     \
                roff = (roff + w16) & rmask16;                                                                                  \
                asm volatile("ld.volatile.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(RN.x), "=r"(RN.y), "=r"(RN.z), "=r"(RN.w) : "r"(ring_s + roff)); \
                KA_SLOT1_DECIDE(act, pos)                                                                                       \
            }                                                                                                                   \
            if (WARP1) __syncwarp(); else __syncthreads();   /* level barrier */                                                \
            pos += w;                                                                                                           \
        }
        // chunks fully inside the ring stages this thread has seen land (a stage = G records = cps chunks + rps records)
        const uint32_t cps = G / w, rps = G - cps * w;
        uint32_t lim_chunks = 0, lim_rem = 0;
        for (uint32_t sdone = 0; sdone < landed; ++sdone) {   // stages observed by the prologue
            lim_chunks += cps; lim_rem += rps;
            if (lim_rem >= w) { lim_rem -= w; ++lim_chunks; }
        }
        while (k < nchunks) {
            // running chunk k prefetches the record of chunk k+1: hand consumed stages back and wait for the next one(s)
            while (landed < nstages && lim_chunks < k + 2) {
                if (tid == 0 && ((released + 1u) << LG) <= (k + 1) * w) {   // every record below (k+1)*w is in registers or done
                    ka_fence_proxy_async();
                    while (((released + 1u) << LG) <= (k + 1) * w) {
                        if (released + NS < nstages_all) issue_stage(released + NS);
                        ++released;
                    }
                }
                ka_mbar_wait(&full[landed & (NS - 1)], (landed / NS) & 1u);
                ++landed;
                lim_chunks += cps; lim_rem += rps;
                if (lim_rem >= w) { lim_rem -= w; ++lim_chunks; }
            }
            // chunks k .. k+n-1 run without a hand-over (after the last stage landed: all of them; the final prefetch reads
            // a stale slot and is ignored)
            const uint32_t n = landed >= nstages ? nchunks - k : min(nchunks, lim_chunks - 1u) - k;
            uint32_t i = 0;
            for (; i + 4 <= n; i += 4) {
                KA_SINGLE_BODY(ra0, rb0)
                KA_SINGLE_BODY(rb0, ra0)
                KA_SINGLE_BODY(ra0, rb0)
                KA_SINGLE_BODY(rb0, ra0)
            }
            for (; i < n; ++i) {
                KA_SINGLE_BODY(ra0, rb0)
                ra0 = rb0;
            }
            k += n;
        }
#undef KA_SINGLE_BODY
    } else if (KIND <= 1) {
        // ---- general chunking (chunk table, or levels wider than the CTA): one body per chunk, unrolled by two ---------------
#define KA_SLOT_BODY(RC, RN)                                                                                                    \
        {                                                                                                                       \
            const uint32_t pos = start + tid;                                                                                   \
            const bool active = pos < end;                                                                                      \
            const uint32_t nstart = end;                                                                                        \
            if (KIND == 0) {                                                                                                    \
                KA_SLOT0_CORE(RC, active, pos)                                                                                  \
                /* next chunk: bounds, stage hand-over, record prefetch: independent of the loads in flight */                \
                const uint32_t nend = next_end(end);                                                                            \
                if (__builtin_expect(nend > limit, 0)) cross_to(end, nend);   /* rare: a new ring stage */                      \
                read_rec(nstart + tid, RN, rb1);                                                                                \
                KA_SLOT0_DECIDE(active, pos)                                                                                    \
                end = nend;                                                                                                     \
            } else {                                                                                                            \
                KA_SLOT1_CORE(RC, active, pos)                                                                                  \
                const uint32_t nend = next_end(end);                                                                            \
                if (__builtin_expect(nend > limit, 0)) cross_to(end, nend);                                                     \
                read_rec(nstart + tid, RN, rb1);                                                                                \
                KA_SLOT1_DECIDE(active, pos)                                                                                    \
                end = nend;                                                                                                     \
            }                                                                                                                   \
            /* level barrier: every counter bump of this chunk is visible before the next chunk reads */                       \
            if (WARP1) __syncwarp(); else __syncthreads();                                                             \
            start = nstart;                                                                                                     \
        }
        while (true) {
            KA_SLOT_BODY(ra0, rb0)
            if (start >= Q) break;
            KA_SLOT_BODY(rb0, ra0)
            if (start >= Q) break;
        }
#undef KA_SLOT_BODY
    } else {
        while (start < Q) {
            const uint32_t pos = start + tid;
            const bool active = pos < end;
            uint4 nb0, nb1;
            (void)pos;
            // ---- rows of 4 / 5..8 replicas: array form, rows written here ---------------------------------------------
            const uint32_t meta = active ? ra1.x : 0u;
            const uint32_t orow = ra1.y;
            const int len = (int)(meta & 15u);
            uint32_t av[RS];  // broker index << 4
            av[0] = (ra0.x & 0xFFFFu) << 4; av[1] = (ra0.x >> 16) << 4; av[2] = (ra0.y & 0xFFFFu) << 4; av[3] = (ra0.y >> 16) << 4;
            if (RS == 8) {
                av[4] = (ra0.z & 0xFFFFu) << 4; av[5] = (ra0.z >> 16) << 4; av[6] = (ra0.w & 0xFFFFu) << 4; av[7] = (ra0.w >> 16) << 4;
            }
            int cv[RS][RS];
#pragma unroll
            for (int i = 0; i < RS; ++i) {
                if (i < len) {
                    const typename C::H h = C::template row<CW>(cbase, ctr8, av[i]);
#pragma unroll
                    for (int v = 0; v < RS; v += 4) {
                        const int4 rw = C::ld4(h, v * 4);
                        cv[i][v] = rw.x; cv[i][v + 1] = rw.y; cv[i][v + 2] = rw.z; cv[i][v + 3] = rw.w;
                    }
                } else {
#pragma unroll
                    for (int v = 0; v < RS; ++v) cv[i][v] = 0;
                }
            }
            const uint32_t nstart = end;
            const uint32_t nend = next_end(end);
            if (nend > limit) cross_to(end, nend);
            read_rec(nstart + tid, nb0, nb1);
            int perm[RS];
#pragma unroll
            for (int i = 0; i < RS; ++i) perm[i] = i;
            if (len > 0) ka_order_generic<RS>(cv, len, meta, perm);
#pragma unroll
            for (int r = 0; r < RS; ++r) {
                if (r < len) {
                    uint32_t ba = 0;
                    int cc = 0;
#pragma unroll
                    for (int q = 0; q < RS; ++q)
                        if (perm[r] == q) { ba = av[q]; cc = cv[q][r]; }
                    C::st(C::template row<CW>(cbase, ctr8, ba), r * 4, cc + 1);  // counter[list[r]][r] += 1 (KAS:254-261)
                    if (r < p.S) p.out[(size_t)orow * p.S + r] = __ldg(&p.broker_id[ba >> 4]);
                } else if (active && r < p.S) {
                    p.out[(size_t)orow * p.S + r] = -1;
                }
            }
            if (active && p.out_len) p.out_len[orow] = len;
            if (NT == 32) __syncwarp(); else __syncthreads();
            start = nstart; end = nend;
            ra0 = nb0; ra1 = nb1;
        }
    }

    // the next chain launch may run its prologue now; its counter load still waits for this grid to complete
    ka_launch_dependents();
    if (!GCTR) {
        if (NT == 32) __syncwarp(); else __syncthreads();
        for (uint32_t i = tid; i < (uint32_t)(CAND ? (int)pin[8] : p.N) * CW; i += NT) ctr8[(i / CW) * KA_MAX_SLOTS + (KIND <= 1 ? KIND : (int)(i % CW))] = ctr[i];
    }
}

// ------------------------------------------------------------------------------------------------
// Emit (rows of <= 3 replicas): ordered record -> broker ids + list length + the slot-2 counters, one thread per schedule
// position, fully parallel; keeps the id lookups and the 4 B/replica output stream off the serial chain.
// ------------------------------------------------------------------------------------------------
// base: the input row of rec[0] and out[0] (part_off counts input rows; 0 but for a cluster of a fleet).
__device__ __forceinline__ void ka_emit3(const uint4* __restrict__ rec, const uint16_t* __restrict__ perm,
                                         const int64_t* __restrict__ part_off, int T, int P, const int32_t* __restrict__ broker_id,
                                         uint32_t Q, int S, int32_t* __restrict__ out, int32_t* __restrict__ out_len,
                                         int32_t* __restrict__ ctr8, uint32_t base = 0) {
    const uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= Q) return;
    const uint4 r = rec[pos];   // ordered by the slot chains: {o0, o1, o2, f}, o_r = broker index << 2
    const int len = (int)(r.w & 3u);
    uint32_t row = pos;
    if (perm) {  // schedule position -> partition row: topic base + ordinal
        int64_t g0;
        if (part_off) {
            int lo = 0, hi = T;  // last topic with part_off[t] <= pos
            while (hi - lo > 1) {
                const int mid = (lo + hi) >> 1;
                if (part_off[mid] <= (int64_t)(base + pos)) lo = mid; else hi = mid;
            }
            g0 = part_off[lo] - base;
        } else {
            g0 = (int64_t)(pos / (uint32_t)P) * P;
        }
        row = (uint32_t)g0 + perm[pos];
    }
    int32_t* o = out + (size_t)row * S;
    o[0] = len > 0 ? __ldg(broker_id + (r.x >> 2)) : -1;
    if (S > 1) o[1] = len > 1 ? __ldg(broker_id + (r.y >> 2)) : -1;
    if (S > 2) o[2] = len > 2 ? __ldg(broker_id + (r.z >> 2)) : -1;
    if (out_len) out_len[row] = len;
    // counter[list[2]][2] += 1 (KAS:254-261): never compared by a row of <= 3 replicas, i.e. a plain commutative sum
    if (len > 2) atomicAdd(ctr8 + (size_t)(r.z >> 2) * KA_MAX_SLOTS + 2, 1);
}

__global__ void __launch_bounds__(256) ka_emit3_kernel(const uint4* __restrict__ rec, const uint16_t* __restrict__ perm,
                                                       const int64_t* __restrict__ part_off, int T, int P,
                                                       const int32_t* __restrict__ broker_id, uint32_t Q, int S, int32_t* __restrict__ out,
                                                       int32_t* __restrict__ out_len, int32_t* __restrict__ ctr8) {
    ka_emit3(rec, perm, part_off, T, P, broker_id, Q, S, out, out_len, ctr8);
}

// Batched solve: blockIdx.y = batch member k. Rows [r0, r0 + Q) of the member's rows (clipped to its window), a sub-block of
// T topics; member k's rows are out + (k * cand_rows + input row) * S (out_len likewise): cand_rows = Q for candidates,
// 0 for the clusters of a fleet, whose rows sit at their input rows. Its counters are its own ctr8. RAGGED: the member's
// whole window (r0 == 0), each schedule position's topic found in the member's part_off[t0 .. t0 + T] as ka_emit3_kernel
// finds it; else dense, P partitions per topic.
template <bool RAGGED = false>
__global__ void __launch_bounds__(256) ka_emit3_candidates_kernel(const KaCandidate* __restrict__ cand, uint32_t r0, int T, int P,
                                                                  const int64_t* __restrict__ part_off, uint32_t Q, int S,
                                                                  int64_t cand_rows, int32_t* __restrict__ out,
                                                                  int32_t* __restrict__ out_len) {
    const KaCandidate& c = cand[blockIdx.y];
    if (c.br.N <= 0 || r0 >= c.Q) return;   // no broker: every topic failed in kernel A, its rows are unspecified
    const uint32_t base = c.row0 + r0;      // input row of the launch's first record of the member
    const int64_t row0 = (int64_t)blockIdx.y * cand_rows + base;
    ka_emit3(reinterpret_cast<const uint4*>(c.out.rec) + base, c.out.perm ? c.out.perm + base : nullptr, RAGGED ? part_off + c.t0 : nullptr,
             RAGGED ? c.T : T, P, c.br.broker_id, min(Q, c.Q - r0), S, out + row0 * S, out_len ? out_len + row0 : nullptr, c.ctr8, base);
}
