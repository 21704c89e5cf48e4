// kassign_score.cuh — movement and balance summary of every member of a batched ragged solve, computed from the emitted rows
// where they already are: every candidate of ka_score_candidates (FLEET = false), every cluster of ka_score_clusters (FLEET =
// true). A sweep or a fleet needs K summaries instead of K copies of the rows.
//
//   ka_score_rows_kernel    one thread per (row, candidate), or per row of a fleet: the row's flags and added / dropped counts
//                           against the current list, warp sums into its member's summary, per-broker sums into [ΣN] arrays
//   ka_score_finish_kernel  one CTA per candidate or cluster: max / min over its brokers and the busiest receiving broker
//
// Everything is integer and every sum commutative, so the results do not depend on the order of the atomics.
#pragma once
#include <climits>

#include "kassign_stage.cuh"
#include "kassign_json.cuh"
#include "../../include/kassign.h"

// A candidate that failed (or has no broker) keeps the zero summary and per-broker entries the host cleared.
__device__ __forceinline__ bool ka_score_ok(const KaCandidate& c) { return c.br.N > 0 && *c.out.err_topic == 0xFFFFFFFFu; }

// Row g's flags and weighted added / dropped counts (row: where its emitted list sits in out / out_len), and its per-broker
// sums into entry bro_off[k] + index of member c's table.
__device__ __forceinline__ void ka_score_row(const KaCandidate& c, const int32_t* bro_off, int k, int64_t row, uint32_t g,
                                             int S, const int32_t* out, const int32_t* out_len,
                                             const int64_t* rep_off, const int32_t* cur,
                                             const int64_t* weight, long long* broker_replicas,
                                             long long* broker_leaders, long long* broker_in, int& changed,
                                             int& moved, int& leader, long long& added, long long& dropped) {
    const int n = out_len[row];
    const int64_t a = rep_off[g];
    const int m = (int)(rep_off[g + 1] - a);
    int nb[3], cb[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        nb[j] = j < n ? out[row * S + j] : 0;
        cb[j] = j < m ? __ldg(cur + a + j) : 0;
    }
    const long long w = weight ? __ldg(weight + g) : 1;
    const KaBrokers br = c.br;   // read once: the atomics below may alias HBM as far as the compiler knows
    const int64_t base = bro_off[k];
    int n_add = 0, n_drop = 0;
    bool diff = n != m;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        if (j < m) {
            bool kept = false;
#pragma unroll
            for (int i = 0; i < 3; ++i) kept |= i < n && nb[i] == cb[j];
            n_drop += !kept;
        }
        if (j < n) {
            bool held = false;
#pragma unroll
            for (int i = 0; i < 3; ++i) held |= i < m && cb[i] == nb[j];
            n_add += !held;
            diff |= j < m && nb[j] != cb[j];
            // the member's id -> index lookup of kernel A, its table read from HBM
            const int64_t e = base + ka_lookup(nb[j], br.blob + br.lut_off, br);
            atomicAdd(reinterpret_cast<unsigned long long*>(broker_replicas + e), (unsigned long long)w);
            if (j == 0) atomicAdd(reinterpret_cast<unsigned long long*>(broker_leaders + e), (unsigned long long)w);
            if (!held) atomicAdd(reinterpret_cast<unsigned long long*>(broker_in + e), (unsigned long long)w);
        }
    }
    changed = diff;
    moved = n_add + n_drop > 0;
    leader = m == 0 || n == 0 || nb[0] != cb[0];
    added = w * n_add;
    dropped = w * n_drop;
}

// FLEET = false: grid (ceil(Q / 256), K). Row g of candidate k is out[(k * Q + g) * S ..] / out_len[k * Q + g].
// FLEET = true: grid (ceil(Q / 256)), Q = ΣP of a fleet. Row g belongs to cluster k with sg.row0[k] <= g < sg.row0[k + 1], and
// sits at its input row; the cluster is live when it is batch member sg.member[k] and that member solved (ka_score_ok). Rows
// of dead clusters add nothing.
// Either way its current list is cur[rep_off[g] .. rep_off[g + 1]), at most S <= 3 long, and ka_score_row scores it; only
// finding the row's member differs between the instances. weight: [Q] or null (1 per row).
// bro_off[k]: member k's (cluster k's) first entry in the per-broker arrays (cand_off of the call); summary: [K].
template <bool FLEET>
__global__ void __launch_bounds__(256) ka_score_rows_kernel(const KaCandidate* __restrict__ cand, const int32_t* __restrict__ bro_off,
                                                            uint32_t Q, int S, const int32_t* __restrict__ out,
                                                            const int32_t* __restrict__ out_len, const int64_t* __restrict__ rep_off,
                                                            const int32_t* __restrict__ cur, const int64_t* __restrict__ weight,
                                                            ka_move_summary* __restrict__ summary, long long* __restrict__ broker_replicas,
                                                            long long* __restrict__ broker_leaders, long long* __restrict__ broker_in,
                                                            const KaJsonSegs sg) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    int k, member;   // the summary the row adds to; the batch member that scores it, -1: the row adds nothing
    int64_t row;
    unsigned grp;    // the lanes that add to summary k
    if constexpr (FLEET) {
        __shared__ int64_t row0[KA_JSON_MAX_SEGS + 1];
        __shared__ int live[KA_JSON_MAX_SEGS];   // cluster k's batch member, -1 = dead
        ka_json_stage_segs(sg, row0, nullptr);
        for (int i = threadIdx.x; i < sg.K; i += blockDim.x) {
            const int m = sg.member[i];
            live[i] = m >= 0 && ka_score_ok(cand[m]) ? m : -1;
        }
        __syncthreads();
        k = g < Q ? ka_json_seg_of(row0, sg.K, g) : -1;
        member = k >= 0 ? live[k] : -1;
        row = g;
        grp = __match_any_sync(KA_FULL, k);   // a warp may span clusters: one group, and one atomic per field, per cluster
    } else {
        k = blockIdx.y;
        if (!ka_score_ok(cand[k])) return;   // CTA-uniform: every lane below reaches the group sums
        member = g < Q ? k : -1;
        row = (int64_t)k * Q + g;
        grp = KA_FULL;
    }
    int changed = 0, moved = 0, leader = 0;
    long long added = 0, dropped = 0;
    if (member >= 0)
        ka_score_row(cand[member], bro_off, k, row, g, S, out, out_len, rep_off, cur, weight, broker_replicas, broker_leaders,
                     broker_in, changed, moved, leader, added, dropped);
    changed = __reduce_add_sync(grp, changed);
    moved = __reduce_add_sync(grp, moved);
    leader = __reduce_add_sync(grp, leader);
    added = ka_group_sum64(added, grp);   // the host holds 3 x the sum of the weights to INT64_MAX
    dropped = ka_group_sum64(dropped, grp);
    if (k >= 0 && (int)(threadIdx.x & 31) == __ffs(grp) - 1) {
        ka_move_summary& s = summary[k];
        auto add = [](int64_t& f, long long v) {
            if (v) atomicAdd(reinterpret_cast<unsigned long long*>(&f), (unsigned long long)v);
        };
        add(s.rows_changed, changed);
        add(s.rows_moved, moved);
        add(s.leaders_changed, leader);
        add(s.replicas_added, added);
        add(s.replicas_dropped, dropped);
    }
}

// grid K, 256 threads: the per-broker extremes of candidate k (FLEET: cluster k, through its batch member sg.member[k]) over all
// N_k of its brokers (brokers left with nothing count), and the busiest receiving broker, the lowest id on ties (indices ascend
// with ids). A failed candidate, or a cluster that is no batch member or failed: zeros, id -1.
template <bool FLEET>
__global__ void __launch_bounds__(256) ka_score_finish_kernel(const KaCandidate* __restrict__ cand, const int32_t* __restrict__ bro_off,
                                                              ka_move_summary* __restrict__ summary,
                                                              const long long* __restrict__ broker_replicas,
                                                              const long long* __restrict__ broker_leaders,
                                                              const long long* __restrict__ broker_in, const KaJsonSegs sg) {
    __shared__ long long sh[8][6];
    const int k = blockIdx.x;
    const KaCandidate* c;
    int n;
    if constexpr (FLEET) {
        const int m = sg.member[k];
        c = m >= 0 ? cand + m : nullptr;
        n = c && ka_score_ok(*c) ? c->br.N : 0;
    } else {
        c = cand + k;
        n = ka_score_ok(*c) ? c->br.N : 0;
    }
    const int64_t base = bro_off[k];
    long long rmax = LLONG_MIN, rmin = LLONG_MAX, lmax = LLONG_MIN, lmin = LLONG_MAX, imax = -1, iarg = INT_MAX;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const long long r = broker_replicas[base + i], l = broker_leaders[base + i], in = broker_in[base + i];
        rmax = max(rmax, r);
        rmin = min(rmin, r);
        lmax = max(lmax, l);
        lmin = min(lmin, l);
        if (in > imax) { imax = in; iarg = i; }   // i ascends: the first maximum is the lowest index
    }
    auto fold = [&](long long orm, long long orn, long long olm, long long oln, long long oim, long long oia) {
        rmax = max(rmax, orm);
        rmin = min(rmin, orn);
        lmax = max(lmax, olm);
        lmin = min(lmin, oln);
        if (oim > imax || (oim == imax && oia < iarg)) { imax = oim; iarg = oia; }
    };
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        fold(__shfl_xor_sync(KA_FULL, rmax, o), __shfl_xor_sync(KA_FULL, rmin, o), __shfl_xor_sync(KA_FULL, lmax, o),
             __shfl_xor_sync(KA_FULL, lmin, o), __shfl_xor_sync(KA_FULL, imax, o), __shfl_xor_sync(KA_FULL, iarg, o));
    const int wid = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
        sh[wid][0] = rmax; sh[wid][1] = rmin; sh[wid][2] = lmax; sh[wid][3] = lmin; sh[wid][4] = imax; sh[wid][5] = iarg;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    for (int v = 1; v < (int)(blockDim.x >> 5); ++v) fold(sh[v][0], sh[v][1], sh[v][2], sh[v][3], sh[v][4], sh[v][5]);
    ka_move_summary& s = summary[k];
    const bool any = n > 0;
    s.max_broker_in = any ? imax : 0;
    s.max_broker_in_id = any && imax > 0 ? __ldg(c->br.broker_id + iarg) : -1;
    s.max_broker_replicas = any ? rmax : 0;
    s.min_broker_replicas = any ? rmin : 0;
    s.max_broker_leaders = any ? lmax : 0;
    s.min_broker_leaders = any ? lmin : 0;
}
