// kassign_waves.cuh — a reassignment cut into waves in which no broker receives more than a budget B (ka_plan_waves).
//
// The rule (include/kassign.h): rows in input order; broker b of the table has open[b] = 1, load[b] = 0. A row with receivers
// (new-list brokers its current list lacks) of weight w takes wave = max over its receivers of (open[b] if load[b] == 0 or
// load[b] + w <= B, else open[b] + 1); then every receiver b either opens that wave (open[b] = wave, load[b] = w) or, already in
// it, adds w. A broker's waves only move forward, so its state is two words.
//
//   ka_wave_rows_kernel     one thread per row: checks, changed flag, receivers as table indices (kernel A's ka_lookup on the
//                           table in HBM), a record per moved row, moved rows per CTA
//   ka_level_scan_kernel    CTA offsets of the moved rows (kassign_order.cuh)
//   ka_wave_compact_kernel  the records of the moved rows, in row order, packed
//   ka_wave_chain_kernel    ONE CTA: the serial rule over the records, in rounds (below); logs every (broker, wave, load) bucket
//   ka_wave_sum_kernel      per wave: rows, rows moved, replicas added
//   ka_wave_peak_kernel     per wave: the largest bucket, then (ID) the lowest broker index among the largest
//
// The chain. Two records depend on each other only through a broker they share, so the chain takes KA_WAVE_CHUNK records at a
// time and decides them in rounds. In a round every pending record claims each of its receivers with an atomicMax of a key
// (round, then the earlier record wins); a record that holds all its claims is the earliest pending record on each of its
// brokers, so every earlier record on them has decided and no other record of the round touches them: it decides and updates
// open / load alone. The earliest pending record always holds its claims, so every round decides at least one record; a record
// decides in round 1 + (the latest round among the earlier records of its chunk that share a broker with it).
//
// The sender budget (SEND, ka_plan_waves_send): the first broker of a moved row's current list sends w x receivers; its index x in
// the send table rides in the record's n word, and the chain keeps its words (open, load, claim) as row N + x, after the N
// brokers' rows. A pending record claims its sender's row with the same key as its receivers' and decides only when it holds
// every claim, so the earliest pending record still decides in every round. A record decides in the round after the latest
// earlier record of its chunk that shares a receiver or its sender with it.
//
// The claim rounds exist once (ka_wave_rounds); each rule's chain passes them its decision.
//
// Everything is integer, and every sum and extreme commutative: the plan does not depend on the order of the atomics.
#pragma once
#include "kassign_common.cuh"
#include "kassign_score.cuh"

#define KA_WAVE_THREADS 512
#define KA_WAVE_PER_THREAD 4
#define KA_WAVE_CHUNK (KA_WAVE_THREADS * KA_WAVE_PER_THREAD)   // records decided together
#define KA_WAVE_SLOT_BITS 11                                   // log2(KA_WAVE_CHUNK)
#define KA_WAVE_MAX_ROUND (1u << (32 - KA_WAVE_SLOT_BITS))      // claim keys are (round << 11) | (CHUNK - 1 - slot)
static_assert(KA_WAVE_CHUNK == 1 << KA_WAVE_SLOT_BITS, "a claim key holds a slot of the chunk");

// A moved row: its input row, its receivers (table indices, 16 bits each, in list order) and its weight. n = the receivers;
// with SEND, bits 16..31 hold the sender's index in the send table (KA_WAVE_NO_SENDER for an empty current list).
struct KaWaveRec {
    int32_t row, n;
    long long w;
    unsigned long long lo, hi;   // receivers 0..3 and 4..7
};
static_assert(sizeof(KaWaveRec) == 32, "two 16-byte loads per record");

// A closed (or, at the end, still open) bucket of incoming load: wave, broker index, load > 0.
struct KaWaveBucket {
    int32_t wave, idx;
    long long load;
};

#define KA_WAVE_NO_SENDER 0xFFFFu

// The sender part of a plan (SEND): the send table id[n] (strictly ascending, n <= 65535), the budget C and the sender bucket
// log.
struct KaWaveSend {
    const int32_t* id;
    int n;
    long long C;
    KaWaveBucket* log;
};

// The meta words of a plan, zeroed by the host but for err_row. Kernels without a sender part never read snd.
struct KaWaveMeta {
    unsigned err_row;   // lowest failing row (unsigned atomicMin, init 0xFFFFFFFF)
    int changed;        // some row changed
    int waves;          // W of the chain (the largest wave of a moved row)
    unsigned nlog;      // buckets logged
    unsigned nslog;     // sender buckets logged
    int bound;          // first fit: Wb (atomicMax)
    KaWaveSend snd;
};

__device__ __forceinline__ uint32_t ka_wave_rcv(const KaWaveRec& r, int j) {
    return (uint32_t)((j < 4 ? r.lo >> (16 * j) : r.hi >> (16 * (j - 4))) & 0xFFFFu);
}

// grid ceil(Q / 256), 256 threads. Row g: new list new_broker[g * S .. + new_len[g]) (S <= 8), current list cur[rep_off[g] ..
// rep_off[g + 1]). Writes nrecv[g] (-1 unchanged, else the receivers), wave[g] for the rows without receivers (0 unchanged, 1
// changed), tmp[g] for a row with receivers, cnt[CTA] = its moved rows. A new list naming a broker twice, or a receiver the
// table lacks, fails the row. SEND: so does a row with receivers whose sender (cur[rep_off[g]]) the send table lacks.
template <bool SEND>
__global__ void __launch_bounds__(256) ka_wave_rows_kernel(const KaBrokers br, uint32_t Q, int S, const int64_t* __restrict__ rep_off,
                                                           const int32_t* __restrict__ cur, const int32_t* __restrict__ new_len,
                                                           const int32_t* __restrict__ new_broker, const int64_t* __restrict__ weight,
                                                           int8_t* __restrict__ nrecv, KaWaveRec* __restrict__ tmp,
                                                           int32_t* __restrict__ wave, int32_t* __restrict__ cnt, KaWaveMeta* __restrict__ meta) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    bool diff = false;
    int k = 0;
    if (g < Q) {
        const int n = new_len[g];
        const int64_t a = rep_off[g];
        const int m = (int)(rep_off[g + 1] - a);
        int nb[KA_MAX_SLOTS];
#pragma unroll
        for (int j = 0; j < KA_MAX_SLOTS; ++j) nb[j] = j < n ? __ldg(new_broker + (int64_t)g * S + j) : 0;
        diff = n != m;
        bool bad = false;
        unsigned long long lo = 0, hi = 0;
        const uint16_t* lut = br.blob + br.lut_off;
#pragma unroll
        for (int j = 0; j < KA_MAX_SLOTS; ++j) {
            if (j < n) {
                bool held = false;
                for (int i = 0; i < m; ++i) held |= __ldg(cur + a + i) == nb[j];
                if (j < m) diff |= __ldg(cur + a + j) != nb[j];
                bool dup = false;
#pragma unroll
                for (int i = 0; i < j; ++i) dup |= nb[i] == nb[j];
                if (!held) {
                    const unsigned long long x = ka_lookup(nb[j], lut, br);
                    bad |= x == KA_DEAD;
                    if (k < 4) lo |= x << (16 * k); else hi |= x << (16 * (k - 4));
                    ++k;
                }
                bad |= dup;
            }
        }
        int n_word = k;
        if constexpr (SEND) {
            if (k > 0) {
                uint32_t sx = KA_WAVE_NO_SENDER;
                if (m > 0) {   // the sender's index: a binary search of the send table
                    const int id = __ldg(cur + a);
                    const KaWaveSend& snd = meta->snd;
                    const int32_t* sid = snd.id;
                    const int ns = snd.n;
                    int l = 0, h = ns;
                    while (l < h) {
                        const int mid = (l + h) >> 1;
                        if (__ldg(sid + mid) < id) l = mid + 1; else h = mid;
                    }
                    if (l < ns && __ldg(sid + l) == id) sx = (uint32_t)l;
                    else bad = true;
                }
                n_word |= (int)(sx << 16);
            }
        }
        if (bad) atomicMin(&meta->err_row, g);
        if (!diff) wave[g] = 0;
        else if (k == 0) wave[g] = 1;
        else tmp[g] = KaWaveRec{(int32_t)g, n_word, weight ? __ldg(weight + g) : 1, lo, hi};
        nrecv[g] = diff ? (int8_t)k : (int8_t)-1;
    }
    const int moved = __syncthreads_count(k > 0);
    if (__syncthreads_or(diff) && threadIdx.x == 0) atomicOr(&meta->changed, 1);
    if (threadIdx.x == 0) cnt[blockIdx.x] = moved;
}

// Same grid as the rows pass: the records of its moved rows to rec[off[CTA] + rank among the CTA's moved rows].
__global__ void __launch_bounds__(256) ka_wave_compact_kernel(uint32_t Q, const int8_t* __restrict__ nrecv, const KaWaveRec* __restrict__ tmp,
                                                              const int32_t* __restrict__ off, KaWaveRec* __restrict__ rec) {
    __shared__ int wsum[8];
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool moved = g < Q && nrecv[g] > 0;
    const unsigned b = __ballot_sync(KA_FULL, moved);
    if (lane == 0) wsum[warp] = __popc(b);
    __syncthreads();
    if (!moved) return;
    int pos = off[blockIdx.x] + __popc(b & ka_lanemask_lt());
    for (int v = 0; v < warp; ++v) pos += wsum[v];
    rec[pos] = tmp[g];
}

// The chains' per-row words: shared memory while they fit (GSTATE = false), else global memory read around L1 (the claims are
// L2 atomics).
template <bool GSTATE, typename T>
__device__ __forceinline__ T ka_wave_ld(const T* p) {
    if constexpr (GSTATE) return __ldcg(p);
    else return *p;
}
template <bool GSTATE, typename T>
__device__ __forceinline__ void ka_wave_st(T* p, T v) {
    if constexpr (GSTATE) __stcg(p, v);
    else *p = v;
}

// Bytes the greedy chain keeps per row (load, open, claim): a broker, or with SEND a sender.
#define KA_WAVE_ROW_BYTES 16

// The receivers of a record (SEND: the n word also holds the sender).
template <bool SEND>
__device__ __forceinline__ int ka_wave_nrcv(const KaWaveRec& r) {
    if constexpr (SEND) return r.n & 0xFFFF;
    else return r.n;
}

// The sender's row (N + its send-table index), or -1 for a record without one or a plan without a sender part.
template <bool SEND>
__device__ __forceinline__ int ka_wave_sender(const KaWaveRec& r, int N) {
    if constexpr (SEND) {
        const uint32_t sx = (uint32_t)r.n >> 16;
        return sx != KA_WAVE_NO_SENDER ? N + (int)sx : -1;
    }
    return -1;
}

// The claim rounds of both chains, run by their ONE CTA of KA_WAVE_THREADS over the M records in rec, with claim[rows] zeroed
// (rows = N + ns: the brokers, then the senders). A record that holds the claims of its k receivers and of its sender's row s
// (-1: none) gets its wave from decide(r, k, s), which also makes the rule's updates. Writes wave[row] of every record and
// returns the largest wave this thread decided.
template <bool GSTATE, bool SEND, typename Decide>
__device__ __forceinline__ int ka_wave_rounds(const KaWaveRec* __restrict__ rec, int M, int N, int rows, unsigned* claim,
                                              int32_t* __restrict__ wave, Decide&& decide) {
    const int tid = threadIdx.x;
    unsigned round = 0;
    int my_max = 0;
    for (int base = 0; base < M; base += KA_WAVE_CHUNK) {
        KaWaveRec r[KA_WAVE_PER_THREAD];
        unsigned pend = 0;
#pragma unroll
        for (int e = 0; e < KA_WAVE_PER_THREAD; ++e) {
            const int i = base + e * KA_WAVE_THREADS + tid;
            if (i < M) {
                r[e] = rec[i];
                pend |= 1u << e;
            } else {
                r[e] = KaWaveRec{0, 0, 0, 0, 0};
            }
        }
        for (;;) {
            // N, opaque to the compiler: each round derives the records' sender rows again rather than holding them in
            // registers across the rounds, where the SEND chains would spill
            int n0 = N;
            asm volatile("" : "+r"(n0));
            if (++round == KA_WAVE_MAX_ROUND) {   // the key's round field is full: clear the claims and count again
                for (int i = tid; i < rows; i += KA_WAVE_THREADS) ka_wave_st<GSTATE>(claim + i, 0u);
                __syncthreads();
                round = 1;
            }
            unsigned key[KA_WAVE_PER_THREAD];
#pragma unroll
            for (int e = 0; e < KA_WAVE_PER_THREAD; ++e) {
                key[e] = round << KA_WAVE_SLOT_BITS | (unsigned)(KA_WAVE_CHUNK - 1 - (e * KA_WAVE_THREADS + tid));
                if (!(pend >> e & 1u)) continue;
                for (int j = 0; j < ka_wave_nrcv<SEND>(r[e]); ++j) atomicMax(claim + ka_wave_rcv(r[e], j), key[e]);
                const int s = ka_wave_sender<SEND>(r[e], n0);
                if (s >= 0) atomicMax(claim + s, key[e]);
            }
            __syncthreads();
#pragma unroll
            for (int e = 0; e < KA_WAVE_PER_THREAD; ++e) {
                if (!(pend >> e & 1u)) continue;
                const int k = ka_wave_nrcv<SEND>(r[e]);
                const int s = ka_wave_sender<SEND>(r[e], n0);
                bool own = s < 0 || ka_wave_ld<GSTATE>(claim + s) == key[e];
                for (int j = 0; j < k; ++j) own &= ka_wave_ld<GSTATE>(claim + ka_wave_rcv(r[e], j)) == key[e];
                if (!own) continue;
                const int v = decide(r[e], k, s);
                wave[r[e].row] = v;
                my_max = max(my_max, v);
                pend &= ~(1u << e);
            }
            if (!__syncthreads_or(pend != 0)) break;
        }
    }
    return my_max;
}

// ONE CTA of KA_WAVE_THREADS. The M = off[nblk] records in rec, the table's N brokers, budget B. Writes wave[row] of every
// record, the bucket log and meta->waves / nlog. The state is load / open / claim [rows = N + ns] in shared memory, or from
// state on (GSTATE). SEND: also the sender rule of meta->snd (budget C), the sender buckets in its log and their count in meta->nslog.
// Does nothing when the rows pass failed a row.
template <bool GSTATE, bool SEND>
__global__ void __launch_bounds__(KA_WAVE_THREADS, 1) ka_wave_chain_kernel(const KaWaveRec* __restrict__ rec, const int32_t* __restrict__ off,
                                                                           int nblk, int N, int rows, long long B, int32_t* __restrict__ wave,
                                                                           unsigned char* state, KaWaveBucket* __restrict__ log,
                                                                           KaWaveMeta* __restrict__ meta) {
    extern __shared__ __align__(16) unsigned char ka_wave_smem[];
    __shared__ unsigned nlog;
    __shared__ int wmax;
    if (*(volatile unsigned*)&meta->err_row != 0xFFFFFFFFu) return;   // CTA-uniform
    long long* load = reinterpret_cast<long long*>(GSTATE ? state : ka_wave_smem);
    int* open = reinterpret_cast<int*>(load + rows);
    unsigned* claim = reinterpret_cast<unsigned*>(open + rows);
    const int tid = threadIdx.x;
    for (int i = tid; i < rows; i += KA_WAVE_THREADS) {
        ka_wave_st<GSTATE>(load + i, 0LL);
        ka_wave_st<GSTATE>(open + i, 1);
        ka_wave_st<GSTATE>(claim + i, 0u);
    }
    if (tid == 0) { nlog = 0; wmax = 0; }
    __syncthreads();
    // a closed or still-open bucket of row x: a broker's to the bucket log, a sender's (snd) to the sender log
    auto put = [&](bool snd, int wv, int x, long long l) {
        if (!snd) {
            const unsigned i = atomicAdd(&nlog, 1u);
            log[i] = KaWaveBucket{wv, x, l};
        } else {
            const unsigned i = atomicAdd(&meta->nslog, 1u);
            meta->snd.log[i] = KaWaveBucket{wv, x - N, l};
        }
    };
    const int my_max = ka_wave_rounds<GSTATE, SEND>(rec, off[nblk], N, rows, claim, wave, [&](const KaWaveRec& r, int k, int s) {
        const long long w = r.w;
        int wv = 0;
        auto want = [&](int x, long long amount, long long cap) {   // the record's wave: the latest any of its rows asks for
            const int o = ka_wave_ld<GSTATE>(open + x);
            const long long l = ka_wave_ld<GSTATE>(load + x);
            wv = max(wv, (l == 0 || l + amount <= cap) ? o : o + 1);
        };
        for (int j = 0; j < k; ++j) want((int)ka_wave_rcv(r, j), w, B);
        if (s >= 0) want(s, w * k, meta->snd.C);
        auto take = [&](int x, long long amount, bool snd) {
            const int o = ka_wave_ld<GSTATE>(open + x);
            const long long l = ka_wave_ld<GSTATE>(load + x);
            if (wv > o) {   // x closes its bucket and opens wave wv
                if (l > 0) put(snd, o, x, l);
                ka_wave_st<GSTATE>(open + x, wv);
                ka_wave_st<GSTATE>(load + x, amount);
            } else {
                ka_wave_st<GSTATE>(load + x, l + amount);
            }
        };
        for (int j = 0; j < k; ++j) take((int)ka_wave_rcv(r, j), w, false);
        if (s >= 0) take(s, w * k, true);
        return wv;
    });
    for (int i = tid; i < rows; i += KA_WAVE_THREADS) {   // the buckets still open
        const long long l = ka_wave_ld<GSTATE>(load + i);
        if (l > 0) put(SEND && i >= N, ka_wave_ld<GSTATE>(open + i), i, l);
    }
    atomicMax(&wmax, my_max);
    __syncthreads();
    if (tid == 0) {
        meta->waves = wmax;
        meta->nlog = nlog;
    }
}

// grid ceil(Q / 256), 256 threads, summary[W] zeroed: every changed row adds to its wave's rows, rows_moved and replicas_added.
// A warp sums each wave among its lanes (ka_group_sum64: a row adds at most 8 x its weight, and the host holds 8 x the sum of
// the weights to INT64_MAX), one atomic per wave and field.
__global__ void __launch_bounds__(256) ka_wave_sum_kernel(uint32_t Q, const int8_t* __restrict__ nrecv, const int32_t* __restrict__ wave,
                                                          const int64_t* __restrict__ weight, ka_wave_summary* __restrict__ summary) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    const int v = g < Q ? wave[g] : 0;
    const int nr = g < Q ? nrecv[g] : -1;
    const long long added = nr > 0 ? (weight ? __ldg(weight + g) : 1) * nr : 0;
    const unsigned grp = __match_any_sync(KA_FULL, v);
    const unsigned rows = __reduce_add_sync(grp, (unsigned)(v > 0));
    const unsigned moved = __reduce_add_sync(grp, (unsigned)(nr > 0));
    const long long sum = ka_group_sum64(added, grp);
    if (v > 0 && (int)(threadIdx.x & 31) == __ffs(grp) - 1) {
        ka_wave_summary& s = summary[v - 1];
        atomicAdd(reinterpret_cast<unsigned long long*>(&s.rows), (unsigned long long)rows);
        if (moved) atomicAdd(reinterpret_cast<unsigned long long*>(&s.rows_moved), (unsigned long long)moved);
        if (sum) atomicAdd(reinterpret_cast<unsigned long long*>(&s.replicas_added), (unsigned long long)sum);
    }
}

// The fields a peak pass fills: the incoming peak of ka_wave_summary over the bucket log, and the outgoing peak of
// ka_wave_send_summary over the sender log.
struct KaWaveInPeak {
    using S = ka_wave_summary;
    static __device__ __forceinline__ int64_t& peak(S& s) { return s.max_broker_in; }
    static __device__ __forceinline__ int64_t& id(S& s) { return s.max_broker_in_id; }
};
struct KaWaveOutPeak {
    using S = ka_wave_send_summary;
    static __device__ __forceinline__ int64_t& peak(S& s) { return s.max_broker_out; }
    static __device__ __forceinline__ int64_t& id(S& s) { return s.max_broker_out_id; }
};

// grid-stride over the n logged buckets, summary zeroed beforehand, into the fields F names. ID = false: peak[wave] = the
// largest bucket of the wave. ID = true (after): id[wave] = N - the lowest index among the buckets equal to that maximum, 0
// when the wave has no bucket (the host turns it into the broker's id, or -1).
template <bool ID, typename F>
__global__ void __launch_bounds__(256) ka_wave_peak_kernel(const KaWaveBucket* __restrict__ log, unsigned n, int N,
                                                           typename F::S* summary) {
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const KaWaveBucket b = log[i];
        typename F::S& s = summary[b.wave - 1];
        if constexpr (!ID) {
            if (b.load > *(volatile long long*)&F::peak(s))   // most buckets lose without an atomic
                atomicMax(reinterpret_cast<unsigned long long*>(&F::peak(s)), (unsigned long long)b.load);
        } else {
            const long long key = N - b.idx;
            if (b.load == F::peak(s) && key > *(volatile long long*)&F::id(s))
                atomicMax(reinterpret_cast<unsigned long long*>(&F::id(s)), (unsigned long long)key);
        }
    }
}

// ---- first fit (KA_WAVE_FIRST_FIT, include/kassign.h) --------------------------------------------------------------------------
// A row with receivers takes the SMALLEST wave v >= 1 in which every receiver's bucket (b, v) is empty or takes w within B, and
// (SEND) its sender's bucket takes a = w x receivers within C. A broker's waves no longer only move forward, so its state is a
// row of loads, one per wave: the table [N + ns][Wb] of int64, the senders' rows after the brokers' (sender x is row N + x).
// Wb bounds W: a wave below a row's is refused only by a bucket with nonzero load, which holds an earlier row sharing a receiver
// or the sender, so with R_b / S_s the moved rows b receives / s sends, W <= Wb = min(M, 1 + max over rows of
// sum over its receivers (R_b - 1) + (S_s - 1)).
//
//   ka_wave_fit_count_kernel  R_b and S_s over the packed records (after the compact pass)
//   ka_wave_fit_bound_kernel  Wb, to the meta words the host reads before it sizes the table
//   ka_wave_fit_chain_kernel  ONE CTA: the claim rounds of ka_wave_rounds, with the first-fit decision
//   ka_wave_fit_log_kernel    every nonzero bucket of the table into the bucket logs, for the peak passes
//
// The chain keeps a hint per row of the table: every wave below it has load >= the budget, so it refuses any row of weight >= 1.
// A row of weight >= 1 starts at the largest hint among its receivers and sender and walks up; a row of weight 0 starts at wave 1.

// Bytes the first-fit chain keeps per table row (claim, hint).
#define KA_WAVE_FIT_ROW_BYTES 8

// Same grid as the rows pass: cnt[N + ns] (zeroed) gets R_b, then S_s at N + s. Does nothing when the rows pass failed a row.
template <bool SEND>
__global__ void __launch_bounds__(256) ka_wave_fit_count_kernel(const KaWaveRec* __restrict__ rec, const int32_t* __restrict__ off, int nblk,
                                                                int N, int* __restrict__ cnt, KaWaveMeta* __restrict__ meta) {
    if (*(volatile unsigned*)&meta->err_row != 0xFFFFFFFFu) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= off[nblk]) return;
    const KaWaveRec r = rec[i];
    for (int j = 0; j < ka_wave_nrcv<SEND>(r); ++j) atomicAdd(cnt + ka_wave_rcv(r, j), 1);
    const int s = ka_wave_sender<SEND>(r, N);
    if (s >= 0) atomicAdd(cnt + s, 1);
}

// Same grid: meta->bound = Wb over the counts of ka_wave_fit_count_kernel.
template <bool SEND>
__global__ void __launch_bounds__(256) ka_wave_fit_bound_kernel(const KaWaveRec* __restrict__ rec, const int32_t* __restrict__ off, int nblk,
                                                                int N, const int* __restrict__ cnt, KaWaveMeta* __restrict__ meta) {
    if (*(volatile unsigned*)&meta->err_row != 0xFFFFFFFFu) return;
    const int M = off[nblk];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned v = 0;
    if (i < M) {
        const KaWaveRec r = rec[i];
        long long x = 0;   // up to 8 x (M - 1) + M - 1: beyond int32 for large M
        for (int j = 0; j < ka_wave_nrcv<SEND>(r); ++j) x += cnt[ka_wave_rcv(r, j)] - 1;
        const int s = ka_wave_sender<SEND>(r, N);
        if (s >= 0) x += cnt[s] - 1;
        v = (unsigned)(1 + min(x, (long long)M - 1));
    }
    v = __reduce_max_sync(KA_FULL, v);
    if ((threadIdx.x & 31) == 0 && v) atomicMax(&meta->bound, (int)v);
}

// ONE CTA of KA_WAVE_THREADS. The M = off[nblk] records in rec, the table's N brokers, budget B, the zeroed table [N + ns][Wb].
// Writes wave[row] of every record and meta->waves. The state is claim / hint [rows = N + ns] in shared memory, or from state
// on (GSTATE). SEND: also the senders' rows and budget C of meta->snd. Does nothing when the rows pass failed a row.
template <bool GSTATE, bool SEND>
__global__ void __launch_bounds__(KA_WAVE_THREADS, 1) ka_wave_fit_chain_kernel(const KaWaveRec* __restrict__ rec, const int32_t* __restrict__ off,
                                                                               int nblk, int N, int rows, long long B, int Wb, int32_t* __restrict__ wave,
                                                                               long long* __restrict__ table, unsigned char* state,
                                                                               KaWaveMeta* __restrict__ meta) {
    extern __shared__ __align__(16) unsigned char ka_wave_smem[];
    __shared__ int wmax;
    if (*(volatile unsigned*)&meta->err_row != 0xFFFFFFFFu) return;   // CTA-uniform
    long long C = 0;
    if constexpr (SEND) C = meta->snd.C;
    unsigned* claim = reinterpret_cast<unsigned*>(GSTATE ? state : ka_wave_smem);
    int* hint = reinterpret_cast<int*>(claim + rows);
    const int tid = threadIdx.x;
    for (int i = tid; i < rows; i += KA_WAVE_THREADS) {
        ka_wave_st<GSTATE>(claim + i, 0u);
        ka_wave_st<GSTATE>(hint + i, 1);
    }
    if (tid == 0) wmax = 0;
    __syncthreads();
    const int my_max = ka_wave_rounds<GSTATE, SEND>(rec, off[nblk], N, rows, claim, wave, [&](const KaWaveRec& r, int k, int s) {
        const long long w = r.w, a = w * k;
        int v = 1;
        if (w > 0) {
            for (int j = 0; j < k; ++j) v = max(v, ka_wave_ld<GSTATE>(hint + ka_wave_rcv(r, j)));
            if (s >= 0) v = max(v, ka_wave_ld<GSTATE>(hint + s));
        }
        for (; v < Wb; ++v) {   // Wb itself always fits (the bound above)
            bool fit = true;
            for (int j = 0; j < k && fit; ++j) {
                const long long l = table[(size_t)ka_wave_rcv(r, j) * Wb + v - 1];
                fit = l == 0 || l + w <= B;
            }
            if (fit && s >= 0) {
                const long long l = table[(size_t)s * Wb + v - 1];
                fit = l == 0 || l + a <= C;
            }
            if (fit) break;
        }
        // add to every bucket, and move each row's hint past the waves that are now full
        auto add = [&](int x, long long amount, long long cap) {
            long long* row = table + (size_t)x * Wb;
            row[v - 1] += amount;
            int h = ka_wave_ld<GSTATE>(hint + x);
            if (h != v) return;
            while (h < Wb && row[h - 1] >= cap) ++h;
            ka_wave_st<GSTATE>(hint + x, h);
        };
        for (int j = 0; j < k; ++j) add((int)ka_wave_rcv(r, j), w, B);
        if (s >= 0) add(s, a, C);
        return v;
    });
    atomicMax(&wmax, my_max);
    __syncthreads();
    if (tid == 0) meta->waves = wmax;
}

// grid-stride over the table [N + ns][Wb]: every bucket with nonzero load to the bucket log (meta->nlog, zeroed) or, a sender's
// row (SEND), to the sender log (its nslog, zeroed) with the send-table index. The peak passes read the logs in any order.
template <bool SEND>
__global__ void __launch_bounds__(256) ka_wave_fit_log_kernel(const long long* __restrict__ table, int Wb, int N, size_t n,
                                                              KaWaveBucket* __restrict__ log, KaWaveMeta* __restrict__ meta) {
    const int lane = threadIdx.x & 31;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t base = (size_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n; base += stride) {   // warp-uniform
        const size_t i = base + lane;
        const long long l = i < n ? table[i] : 0;
        const int x = (int)(i / (size_t)Wb);
        const int v = (int)(i % (size_t)Wb) + 1;
        const bool in = l > 0 && x < N;
        const unsigned mi = __ballot_sync(KA_FULL, in);
        unsigned at = 0;
        if (lane == 0 && mi) at = atomicAdd(&meta->nlog, (unsigned)__popc(mi));
        at = __shfl_sync(KA_FULL, at, 0) + __popc(mi & ka_lanemask_lt());
        if (in) log[at] = KaWaveBucket{v, x, l};
        if constexpr (SEND) {
            const bool out = l > 0 && x >= N;
            const unsigned mo = __ballot_sync(KA_FULL, out);
            unsigned so = 0;
            if (lane == 0 && mo) so = atomicAdd(&meta->nslog, (unsigned)__popc(mo));
            so = __shfl_sync(KA_FULL, so, 0) + __popc(mo & ka_lanemask_lt());
            if (out) meta->snd.log[so] = KaWaveBucket{v, x - N, l};
        }
    }
}
