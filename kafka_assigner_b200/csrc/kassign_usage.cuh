// kassign_usage.cuh — every broker's disk usage across a wave plan (ka_wave_broker_usage): what it holds before the plan, its
// peak and the wave of the peak, what it holds after, and the first wave in which it is over its capacity.
//
// The rule (include/kassign.h): a receiver of a row holds the new copy from the start of the row's wave v, a dropper frees its
// copy once wave v has ended. So a row of weight w with wave v > 0 is an EVENT (broker, v, +w) per receiver and (broker, v + 1,
// -w) per distinct dropper, and usage(v) is before + the sum of the broker's events with a wave <= v. The events are sparse: their
// number is bounded by Q x stride + rep_off[Q], whatever the number of waves is.
//
//   ka_usage_rows_kernel     one thread per row: checks, before[] (warp-aggregated 64-bit atomics), the row's events appended
//                            to the event list (one atomic per warp: the list's order is arbitrary, the sort below fixes it)
//   ka_usage_sort_hist_kernel    per tile of events: how many have each value of the pass's 8-bit digit
//   ka_level_scan_kernel         (digit, tile) offsets (kassign_order.cuh)
//   ka_usage_sort_scatter_kernel the tile's events to their digit's range, in tile order (a stable LSD radix pass). The passes
//                                take the wave's digits first, then the broker index's: the events end grouped by broker, in
//                                wave order inside a broker.
//   ka_usage_broker_kernel   one warp per table broker: its segment in wave order, 32 events at a time with a carried prefix
//
// Everything is integer and every sum is of the same terms whatever the order: the report does not depend on the order of the
// atomics or of the unsorted event list.
#pragma once
#include <climits>

#include "kassign_common.cuh"
#include "../../include/kassign.h"

// One event: from wave `wave` on, broker index `idx` holds w more (w < 0: a freed copy). Sorted by the 64-bit key
// idx << 32 | wave.
struct __align__(16) KaUseEvent {
    uint32_t wave, idx;
    long long w;
};
static_assert(sizeof(KaUseEvent) == 16, "one 16-byte load per event");

__device__ __forceinline__ unsigned long long ka_usage_key(const KaUseEvent& e) {
    return (unsigned long long)e.idx << 32 | e.wave;
}

struct KaUsageMeta {
    unsigned err_row;   // lowest failing row (unsigned atomicMin, init 0xFFFFFFFF)
    unsigned nev;       // events appended
};

// Index of `id` in the ascending table id[n], or -1.
__device__ __forceinline__ int ka_usage_find(const int32_t* __restrict__ id, int n, int x) {
    int l = 0, h = n;
    while (l < h) {
        const int mid = (l + h) >> 1;
        if (__ldg(id + mid) < x) l = mid + 1; else h = mid;
    }
    return l < n && __ldg(id + l) == x ? l : -1;
}

// Adds v >= 0 to sum[idx] for every lane with idx >= 0: lanes with the same index add their sum with one atomic. All lanes of
// the warp take part.
__device__ __forceinline__ void ka_usage_add(long long* sum, int idx, long long v) {
    const unsigned grp = __match_any_sync(KA_FULL, idx);
    const long long s = ka_group_sum64(v, grp);
    if (idx >= 0 && (int)(threadIdx.x & 31) == __ffs(grp) - 1)
        atomicAdd(reinterpret_cast<unsigned long long*>(sum + idx), (unsigned long long)s);
}

// grid ceil(Q / 256) (at least 1), 256 threads. Row g: current list cur[rep_off[g] .. rep_off[g + 1]), new list new_broker[g * S ..
// + new_len[g]) (S <= 8), weight w (null: 1), wave[g] >= 0. Table id[n]. A new list naming a broker twice, or a receiver of a row
// with wave > 0 that the table lacks, fails the row. Adds w to before[i] for every distinct table broker i of the current list,
// and appends the events of a row with wave > 0 to ev (meta->nev counts them). Appends nothing once some row has failed.
__global__ void __launch_bounds__(256) ka_usage_rows_kernel(uint32_t Q, int S, const int64_t* __restrict__ rep_off,
                                                            const int32_t* __restrict__ cur, const int32_t* __restrict__ new_len,
                                                            const int32_t* __restrict__ new_broker, const int64_t* __restrict__ weight,
                                                            const int32_t* __restrict__ wave, const int32_t* __restrict__ id, int n,
                                                            long long* __restrict__ before, KaUseEvent* __restrict__ ev,
                                                            KaUsageMeta* __restrict__ meta) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const bool live = g < Q;
    int nl = 0, m = 0, v = 0;
    int64_t a = 0;
    long long w = 0;
    if (live) {
        nl = new_len[g];
        a = rep_off[g];
        m = (int)(rep_off[g + 1] - a);
        v = wave[g];
        w = weight ? __ldg(weight + g) : 1;
    }
    int nb[KA_MAX_SLOTS];
#pragma unroll
    for (int j = 0; j < KA_MAX_SLOTS; ++j) nb[j] = j < nl ? __ldg(new_broker + (int64_t)g * S + j) : 0;
    // the receivers (table indices, 16 bits per position of the new list, KA_DEAD where none) and the checks
    bool bad = false;
    unsigned long long rlo = ~0ull, rhi = ~0ull;
    int k = 0;
#pragma unroll
    for (int j = 0; j < KA_MAX_SLOTS; ++j) {
        if (j < nl) {
            bool held = false, dup = false;
            for (int i = 0; i < m; ++i) held |= __ldg(cur + a + i) == nb[j];
#pragma unroll
            for (int i = 0; i < j; ++i) dup |= nb[i] == nb[j];
            bad |= dup;
            if (!held && v > 0) {
                const int x = ka_usage_find(id, n, nb[j]);
                bad |= x < 0;
                const unsigned long long f = (unsigned long long)(x & 0xFFFF) << (16 * (j & 3));
                if (j < 4) rlo &= ~(0xFFFFull << (16 * j)) | f; else rhi &= ~(0xFFFFull << (16 * (j - 4))) | f;
                ++k;
            }
        }
    }
    if (bad) atomicMin(&meta->err_row, g);
    // before[] and the droppers: the distinct table brokers of the current list, one position at a time across the warp
    int drop = 0;
    const int mmax = __reduce_max_sync(KA_FULL, (unsigned)m);
    for (int i = 0; i < mmax; ++i) {
        int x = -1;
        bool kept = true;
        if (i < m) {
            const int b = __ldg(cur + a + i);
            bool first = true;
            for (int h = 0; h < i; ++h) first &= __ldg(cur + a + h) != b;
            if (first) x = ka_usage_find(id, n, b);
            kept = false;
#pragma unroll
            for (int j = 0; j < KA_MAX_SLOTS; ++j) kept |= j < nl && nb[j] == b;
        }
        ka_usage_add(before, x, x >= 0 ? w : 0);
        drop += x >= 0 && !kept && v > 0;
    }
    // the events: k receivers at wave v, drop droppers at wave v + 1; one slot range per warp
    const int mine = bad ? 0 : k + drop;
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(KA_FULL, incl, o);
        if (lane >= o) incl += y;
    }
    const int tot = __shfl_sync(KA_FULL, incl, 31);
    unsigned at = 0;
    if (lane == 31 && tot > 0) at = atomicAdd(&meta->nev, (unsigned)tot);
    at = __shfl_sync(KA_FULL, at, 31) + (unsigned)(incl - mine);
    if (mine == 0) return;
#pragma unroll
    for (int j = 0; j < KA_MAX_SLOTS; ++j) {
        const uint32_t x = (uint32_t)((j < 4 ? rlo >> (16 * j) : rhi >> (16 * (j - 4))) & 0xFFFFu);
        if (x != KA_DEAD) ev[at++] = KaUseEvent{(uint32_t)v, x, w};
    }
    for (int i = 0; i < m && drop > 0; ++i) {
        const int b = __ldg(cur + a + i);
        bool first = true, kept = false;
        for (int h = 0; h < i; ++h) first &= __ldg(cur + a + h) != b;
#pragma unroll
        for (int j = 0; j < KA_MAX_SLOTS; ++j) kept |= j < nl && nb[j] == b;
        const int x = first && !kept ? ka_usage_find(id, n, b) : -1;
        if (x >= 0) {
            ev[at++] = KaUseEvent{(uint32_t)v + 1u, (uint32_t)x, -w};
            --drop;
        }
    }
}

// One radix pass over the ne events of in, by the digit (key >> shift) & 255. Tile b owns events [b * tile, (b + 1) * tile).
struct KaUsageSort {
    const KaUseEvent* in;
    uint32_t ne;
    int shift;
    uint32_t tile;
    int ntiles;
};

__device__ __forceinline__ int ka_usage_digit(const KaUsageSort& p, const KaUseEvent& e) {
    return (int)(ka_usage_key(e) >> p.shift) & (KA_RADIX_DIGITS - 1);
}

// grid ntiles, 256 threads: hist[digit * ntiles + tile] = the tile's events with that digit.
__global__ void __launch_bounds__(256) ka_usage_sort_hist_kernel(const KaUsageSort p, int32_t* __restrict__ hist) {
    __shared__ int h[KA_RADIX_DIGITS];
    h[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t lo = (uint64_t)blockIdx.x * p.tile;
    const uint32_t hi = (uint32_t)min((uint64_t)p.ne, lo + p.tile);
    for (uint64_t i = lo + threadIdx.x; i < hi; i += 256) atomicAdd(&h[ka_usage_digit(p, p.in[i])], 1);   // a count: any order
    __syncthreads();
    hist[threadIdx.x * p.ntiles + blockIdx.x] = h[threadIdx.x];
}

// Same grid: off = the exclusive scan of hist. Event i of the tile goes to out[off[digit][tile] + its rank among the tile's events
// of that digit]. The tile is taken 256 events at a time; in a round a lane ranks itself among the lanes of its warp with the
// same digit (match_any, lanes in event order), then behind the earlier warps' and the earlier rounds' events of that digit.
__global__ void __launch_bounds__(256) ka_usage_sort_scatter_kernel(const KaUsageSort p, const int32_t* __restrict__ off,
                                                                    KaUseEvent* __restrict__ out) {
    __shared__ int base[KA_RADIX_DIGITS];
    __shared__ int wcnt[8][KA_RADIX_DIGITS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    base[threadIdx.x] = off[threadIdx.x * p.ntiles + blockIdx.x];
    const uint64_t lo = (uint64_t)blockIdx.x * p.tile;
    const uint32_t hi = (uint32_t)min((uint64_t)p.ne, lo + p.tile);
    for (uint64_t r0 = lo; r0 < hi; r0 += 256) {   // CTA-uniform
#pragma unroll
        for (int w = 0; w < 8; ++w) wcnt[w][threadIdx.x] = 0;
        const uint64_t i = r0 + threadIdx.x;
        const bool item = i < hi;
        KaUseEvent e{};
        int digit = -1;
        if (item) {
            e = p.in[i];
            digit = ka_usage_digit(p, e);
        }
        const unsigned same = __match_any_sync(KA_FULL, digit);
        __syncthreads();
        if (item && lane == __ffs(same) - 1) wcnt[warp][digit] = __popc(same);
        __syncthreads();
        if (item) {
            int pos = base[digit] + __popc(same & ka_lanemask_lt());
            for (int w = 0; w < warp; ++w) pos += wcnt[w][digit];
            out[pos] = e;
        }
        __syncthreads();
        int s = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) s += wcnt[w][threadIdx.x];
        base[threadIdx.x] += s;   // column threadIdx.x is this thread's alone until the next round's counts
    }
}

// The 64-bit maximum of (val, key) pairs over the warp, in every lane: the larger val, the larger key among equal vals.
__device__ __forceinline__ void ka_usage_warp_max(long long& val, long long& key) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const long long v2 = __shfl_xor_sync(KA_FULL, val, o), k2 = __shfl_xor_sync(KA_FULL, key, o);
        if (v2 > val || (v2 == val && k2 > key)) { val = v2; key = k2; }
    }
}

// grid ceil(n / 8) (at least 1), 256 threads: warp i reports table broker i < n from the ne events of ev, sorted by (index,
// wave). base / cap: null = 0 / no capacity. W = the plan's largest wave: events at W + 1 (the drops of wave W) count for
// `after` only.
__global__ void __launch_bounds__(256) ka_usage_broker_kernel(const KaUseEvent* __restrict__ ev, uint32_t ne, int n, int W,
                                                              const long long* __restrict__ before, const int64_t* __restrict__ base,
                                                              const int64_t* __restrict__ cap, ka_broker_usage* __restrict__ usage) {
    const int i = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= n) return;   // warp-uniform
    // the segment [s, e) of broker i: two binary searches over the sorted indices
    auto lower = [&](uint32_t x) {
        uint32_t l = 0, h = ne;
        while (l < h) {
            const uint32_t mid = (l + h) >> 1;
            if (ev[mid].idx < x) l = mid + 1; else h = mid;
        }
        return l;
    };
    const uint32_t s = lower((uint32_t)i), e = lower((uint32_t)i + 1);
    const long long b0 = before[i] + (base ? base[i] : 0);
    const long long c = cap ? cap[i] : LLONG_MAX;
    long long run = b0, peak = b0;
    int peak_wave = 0, over = cap && b0 > c ? 0 : -1;
    for (uint32_t k0 = s; k0 < e; k0 += 32) {
        const uint32_t k = k0 + lane;
        const bool in = k < e;
        const KaUseEvent x = in ? ev[k] : KaUseEvent{0xFFFFFFFFu, 0u, 0};
        // the next event's wave: this lane closes its wave when the next event is of another wave (or of another broker)
        const uint32_t nxt = k + 1 < e ? __ldg(&ev[k + 1].wave) : 0xFFFFFFFFu;
        long long pre = x.w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long y = __shfl_up_sync(KA_FULL, pre, o);
            if (lane >= o) pre += y;
        }
        const long long val = run + pre;
        const bool point = in && nxt != x.wave && x.wave <= (uint32_t)W;   // usage(x.wave), for a wave of the plan
        // the largest point of the 32, the lowest wave among equals; an earlier chunk's peak keeps a tie
        long long pv = point ? val : LLONG_MIN, pk = point ? -(long long)x.wave : LLONG_MIN;
        ka_usage_warp_max(pv, pk);
        if (pv > peak) {
            peak = pv;
            peak_wave = (int)-pk;
        }
        if (over < 0) {
            const unsigned hit = __ballot_sync(KA_FULL, point && val > c);
            if (hit) over = (int)__shfl_sync(KA_FULL, x.wave, __ffs(hit) - 1);
        }
        run += __shfl_sync(KA_FULL, pre, 31);
    }
    if (lane == 0) usage[i] = ka_broker_usage{b0, peak, peak_wave, run, over};
}
