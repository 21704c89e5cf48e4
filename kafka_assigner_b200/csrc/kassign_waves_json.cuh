// kassign_waves_json.cuh — one reassignment document per wave of a wave plan (ka_plan_waves_json), built on the device from the
// rows the plan left there, so that only TEXT crosses PCIe.
//
// A wave's rows are scattered over the whole input and there may be as many waves as changed rows, so the documents are not
// segments of the input. The changed rows are first grouped by wave, stably (perm = the changed rows ordered by (wave, row)), and
// the document frame is folded into the rows: the first row of a wave carries {"partitions":[ in place of its leading comma, the
// last one also ],"version":1}. The whole output is then ONE concatenation of the grouped rows' texts, and document v starts
// where the first row of wave v + 1 does.
//
//   ka_wave_sort_hist_kernel     per tile of rows: how many keys have each value of the pass's 8-bit digit
//   ka_level_scan_kernel         (digit, tile) offsets (kassign_order.cuh); their total is M, the changed rows
//   ka_wave_sort_scatter_kernel  the tile's rows to their digit's range, in row order (a stable LSD radix pass). The first pass
//                                reads the rows 0..Q-1 themselves and drops wave 0, so it also compacts.
//   ka_wave_doc_len_kernel       text bytes of every grouped row + per-CTA sums
//   ka_wave_doc_scan_kernel      ONE CTA: 64-bit text offsets of the CTAs, and the total
//   ka_wave_doc_write_kernel     the text (through the JSON passes' shared-memory stage) and doc_off[0..W]
//
// A size limit L (ka_plan_waves_json_parts) cuts every wave into PARTS, runs of consecutive grouped rows, greedily: a row joins
// its wave's current part while that part's document stays <= L. With c_i = a record's bytes + 1 (its comma) and S the 64-bit
// exclusive prefix of c over the grouped positions, positions i..j-1 of one wave make a document of S[j] - S[i] + 28 bytes.
//
//   ka_wave_part_len_kernel      c_i, per-CTA sums, the first position of every wave, the wave starts as part starts
//   ka_wave_doc_scan_kernel      ONE CTA: the CTA sums to offsets
//   ka_wave_part_prefix_kernel   S[0..M]
//   ka_wave_part_next_kernel     J_0[i] = where a part opened at i ends (binary search over S within the wave; M = the wave's
//                                end); a record that alone exceeds L reports its row; the most rows of a wave
//   ka_wave_part_jump_kernel     J_k = J_{k-1} o J_{k-1}, k = 1 .. K-1, with 2^K >= the most rows of a wave
//   ka_wave_part_mark_kernel     k = K-1 .. 0: every part start i marks J_k[i]. Starting from the wave starts, level k adds the
//                                starts 2^k parts further on, so after level 0 every start is marked. A mark only ever sets a
//                                start, and every start is set by some level: the flags do not depend on the order of stores.
// The text passes then run with PARTS = true: the frame goes at part boundaries and doc_off is indexed by part. They add the
// parts starting in every CTA, and the scan numbers the parts (D, the parts of all waves).
//
// The rollback documents (ka_plan_waves_json_parts_rollback) print every part's rows with their CURRENT lists
// (ka_json_back_len / ka_json_back_put). The paired cut takes the rollback record's c'_i beside c_i and its prefix R beside S:
// positions i..j-1 of one wave make a part iff both S[j] - S[i] and R[j] - R[i] are <= L - 28. The part passes' BACK = true
// instances carry R (the pair scan ka_wave_part_scan_kernel<2> takes the place of ka_wave_doc_scan_kernel); the jump and mark
// passes are the same. The rollback text is then one more length / scan / write trio (BACK = true, over the same positions and
// part starts), into its own buffer, with the frame {"version":1,"partitions":[ ... ]}.
//
// The part caps (ka_ctx_set_part_caps) bound what one part holds: at most Lr rows, and at most Lx of data, a_i = w[g] x the
// receivers of row g = perm[i] (0 for a row that only reorders), unless the part is a single row. The CAPS = true instances of
// the length, prefix and next passes carry A, the 64-bit exclusive prefix of a, beside S (and R): the length pass writes a_i
// and its CTA sums, the one-CTA scan takes them as one more array (ka_wave_part_scan_kernel<2> or <3>), the prefix pass turns
// a_i into A[i], and the next pass ends its search at i + Lr and tests A[j] - A[i] <= Lx beside the bytes. j = i + 1 is never
// tested: a single row always makes a part, so only the byte limit can refuse a row. The launches are those of the uncapped
// call.
//
// A pass ranks a row by counting, never by the order of atomics: the text depends on the input alone.
#pragma once
#include "kassign_json.cuh"
#include "kassign_waves.cuh"

// One radix pass over the keys wave[g] >> shift. in == null: the items are the rows 0..Q-1 (first pass); else the *n_ptr rows
// in[]. A row of wave 0 is no item. Tile b owns items [b * tile, (b + 1) * tile).
struct KaWaveSort {
    const int32_t* wave;
    const int32_t* in;
    uint32_t Q;
    const int32_t* n_ptr;
    int shift;
    uint32_t tile;
    int ntiles;
};

__device__ __forceinline__ bool ka_wave_sort_item(const KaWaveSort& p, uint32_t i, uint32_t hi, int32_t& g, int& digit) {
    if (i >= hi) return false;
    g = p.in ? p.in[i] : (int32_t)i;
    const int v = p.wave[g];
    digit = (v >> p.shift) & (KA_RADIX_DIGITS - 1);
    return v > 0;
}

// grid ntiles, 256 threads: hist[digit * ntiles + tile] = the tile's items with that digit.
__global__ void __launch_bounds__(256) ka_wave_sort_hist_kernel(const KaWaveSort p, int32_t* __restrict__ hist) {
    __shared__ int h[KA_RADIX_DIGITS];
    h[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t n = p.in ? (uint32_t)*p.n_ptr : p.Q;
    const uint64_t lo = (uint64_t)blockIdx.x * p.tile;
    const uint32_t hi = (uint32_t)min((uint64_t)n, lo + p.tile);
    for (uint64_t i = lo + threadIdx.x; i < hi; i += 256) {
        int32_t g;
        int digit;
        if (ka_wave_sort_item(p, (uint32_t)i, hi, g, digit)) atomicAdd(&h[digit], 1);   // a count: any order gives it
    }
    __syncthreads();
    hist[threadIdx.x * p.ntiles + blockIdx.x] = h[threadIdx.x];
}

// Same grid: off = the exclusive scan of hist. Item i of the tile goes to out[off[digit][tile] + its rank among the tile's items
// of that digit]. The tile is taken 256 items at a time; in a round a lane ranks itself among the lanes of its warp with the
// same digit (match_any, lanes in item order), then behind the earlier warps' and the earlier rounds' items of that digit.
__global__ void __launch_bounds__(256) ka_wave_sort_scatter_kernel(const KaWaveSort p, const int32_t* __restrict__ off,
                                                                   int32_t* __restrict__ out) {
    __shared__ int base[KA_RADIX_DIGITS];
    __shared__ int wcnt[8][KA_RADIX_DIGITS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    base[threadIdx.x] = off[threadIdx.x * p.ntiles + blockIdx.x];
    const uint32_t n = p.in ? (uint32_t)*p.n_ptr : p.Q;
    const uint64_t lo = (uint64_t)blockIdx.x * p.tile;
    const uint32_t hi = (uint32_t)min((uint64_t)n, lo + p.tile);
    for (uint64_t r0 = lo; r0 < hi; r0 += 256) {   // CTA-uniform
#pragma unroll
        for (int w = 0; w < 8; ++w) wcnt[w][threadIdx.x] = 0;
        int32_t g = 0;
        int digit = 0;
        const bool item = ka_wave_sort_item(p, (uint32_t)(r0 + threadIdx.x), hi, g, digit);
        const unsigned same = __match_any_sync(KA_FULL, item ? digit : -1);
        __syncthreads();
        if (item && lane == __ffs(same) - 1) wcnt[warp][digit] = __popc(same);
        __syncthreads();
        if (item) {
            int pos = base[digit] + __popc(same & ka_lanemask_lt());
            for (int w = 0; w < warp; ++w) pos += wcnt[w][digit];
            out[pos] = g;
        }
        __syncthreads();
        int s = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) s += wcnt[w][threadIdx.x];
        base[threadIdx.x] += s;   // column threadIdx.x is this thread's alone until the next round's counts
    }
}

// The text passes. Grouped position i < M = *n_rows holds row perm[i]; p describes the run's rows (row0 = 0, so its row q is the
// run-wide row g: p.out / p.out_len are the proposed lists, p.rowlen is indexed by POSITION here). The grids cover Q rows, M is
// only known on the device: the CTAs beyond it do nothing.
struct KaWaveDocs {
    KaJsonParams p;
    const int32_t* wave;                 // [Q]
    const int32_t* perm;                 // [M]
    const int32_t* n_rows;               // M
    unsigned long long* blockoff;        // [ceil(Q / 256)] text bytes of every CTA, then (scan) its text offset
    unsigned long long* doc_off;         // [W + 1] out, with PARTS [D + 1]
};

// What the text passes read and write only with PARTS = true, which places the frame at part boundaries instead of wave
// boundaries. A separate (last) kernel argument, so that the PARTS = false instances keep the parameter layout of KaWaveDocs.
struct KaWaveDocParts {
    const uint8_t* start;                // [M] 1 where a part starts
    int* part_cnt;                       // [ceil(Q / 256)] parts starting in every CTA, then (scan) the parts before it
    int32_t* doc_wave;                   // [D] out: the wave of every part
};

// What the passes read and write only for the rollback documents (BACK = true): the current lists, and the rollback side's row
// bytes, CTA sums / offsets and (part passes) prefix R. A separate (last) kernel argument, like KaWaveDocParts.
struct KaWaveBack {
    const int64_t* rep_off;              // [Q + 1]
    const int32_t* cur;                  // [rep_off[Q]]
    uint32_t* rowlen;                    // [M] c'_i in the part passes, then the rollback text bytes of every position
    unsigned long long* blockoff;        // [ceil(Q / 256)] CTA sums, then (scan) their offsets
    unsigned long long* R;               // [M + 1] the part passes' prefix of c'
};

// What the part passes read and write only under the part caps (CAPS = true). A separate (last) kernel argument, like
// KaWaveBack.
struct KaWaveCaps {
    const int8_t* nrecv;                 // [Q] the plan's receivers of every row (-1 for an unchanged row)
    const int64_t* weight;               // [Q], or null: 1 per row
    unsigned long long* blockoff;        // [ceil(Q / 256)] the CTA sums of a, then (scan) their offsets
    unsigned long long* A;               // [M + 1] a_i (length pass), then (prefix pass) the exclusive prefix of a
    unsigned long long rows;             // Lr, or 2^32 without a row cap
    unsigned long long in;               // Lx, or ~0 without a data cap
};

// ka_cta256_prefix over 64-bit values: this thread's offset in the CTA's sum, and (total) that sum, in every thread.
__device__ __forceinline__ unsigned long long ka_cta256_prefix64(unsigned long long n, unsigned long long& total) {
    __shared__ unsigned long long wsum[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long x = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(KA_FULL, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    unsigned long long woff = 0;
    total = 0;
    for (int i = 0; i < 8; ++i) { if (i < warp) woff += wsum[i]; total += wsum[i]; }
    return woff + x - n;
}

// Row, wave and place in its document of grouped position i.
template <bool PARTS>
__device__ __forceinline__ void ka_wave_doc_row(const KaWaveDocs& d, const KaWaveDocParts& pd, uint32_t i, uint32_t M, uint32_t& g, int& v,
                                                bool& first, bool& last) {
    g = (uint32_t)d.perm[i];
    v = d.wave[g];
    if constexpr (PARTS) {
        first = pd.start[i];
        last = i + 1 == M || pd.start[i + 1];
    } else {
        first = i == 0 || d.wave[d.perm[i - 1]] != v;
        last = i + 1 == M || d.wave[d.perm[i + 1]] != v;
    }
}

// grid ceil(Q / 256), 256 threads. BACK (with PARTS): the rollback text, whose parts the PARTS = true pass has counted already.
template <bool PARTS, bool BACK>
__global__ void __launch_bounds__(256) ka_wave_doc_len_kernel(const KaWaveDocs d, const KaWaveDocParts pd, const KaWaveBack bk) {
    const uint32_t M = (uint32_t)*d.n_rows;
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    uint32_t n = 0;
    bool opens = false;
    if (i < M) {
        uint32_t g;
        int v;
        bool first, last;
        ka_wave_doc_row<PARTS>(d, pd, i, M, g, v, first, last);
        if constexpr (BACK)
            n = (first ? KA_BACK_HEAD_LEN : 0u) + ka_json_back_len(d.p, bk.rep_off, bk.cur, g, !first) + (last ? KA_BACK_TAIL_LEN : 0u);
        else
            n = (first ? KA_JSON_HEAD_LEN : 0u) + ka_json_row_len(d.p, g, !first) + (last ? KA_JSON_TAIL_LEN : 0u);
        d.p.rowlen[i] = n;
        opens = first;
    }
    const unsigned long long bytes = ka_cta256_sum(n);
    if (threadIdx.x == 0) d.blockoff[blockIdx.x] = bytes;
    if constexpr (PARTS && !BACK) {
        const int parts = __syncthreads_count(opens);
        if (threadIdx.x == 0) pd.part_cnt[blockIdx.x] = parts;
    }
}

// ONE CTA of 1024: v[0..n) to its exclusive scan in place, *total = the sum. 64-bit throughout: 8 bytes per 256 rows lift the
// 4 GiB limit a fragment of ka_json_scan_kernel has. PARTS: cnt[0..n) likewise, total[1] = D.
template <bool PARTS>
__global__ void __launch_bounds__(1024) ka_wave_doc_scan_kernel(unsigned long long* __restrict__ v, int n, unsigned long long* __restrict__ total,
                                                                int* __restrict__ cnt) {
    const unsigned long long bytes = ka_cta_scan(v, v, n, 0ull);
    if (threadIdx.x == 0) *total = bytes;
    if constexpr (PARTS) {
        const int parts = ka_cta_scan(cnt, cnt, n, 0);
        if (threadIdx.x == 0) total[1] = (unsigned long long)parts;
    }
}

// grid ceil(Q / 256), 256 threads, KA_JSON_SMEM_BYTES + 16 of dynamic shared memory. Every grouped row writes its text at its
// final position, the 256 rows of a CTA through the shared-memory stage of the JSON passes. The frame travels with the rows,
// so a CTA that spans many waves is staged like any other. The first row of wave v writes doc_off[v - 1], the last row of all
// doc_off[W]; PARTS: the first row of part r writes doc_off[r] and doc_wave[r], the last row of all doc_off[D]. BACK: the
// rollback text, whose doc_off is back_off and which writes no doc_wave. Nothing is written when the text exceeds p.cap.
template <bool PARTS, bool BACK>
__global__ void __launch_bounds__(256) ka_wave_doc_write_kernel(const KaWaveDocs d, const unsigned long long* __restrict__ total,
                                                                const KaWaveDocParts pd, const KaWaveBack bk) {
    extern __shared__ __align__(16) unsigned char ka_jsmem[];
    const uint32_t M = (uint32_t)*d.n_rows;
    if (*total > d.p.cap || blockIdx.x * 256u >= M) return;   // CTA-uniform
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    const uint32_t n = i < M ? d.p.rowlen[i] : 0u;
    uint32_t bt;
    const uint32_t loc = ka_cta256_prefix(n, bt);           // my row inside the CTA's text
    uint32_t part = 0;                                      // PARTS: my part, when I open one
    if constexpr (PARTS) {
        __shared__ int wparts[8];
        const unsigned opens = __ballot_sync(KA_FULL, i < M && pd.start[i]);
        if ((threadIdx.x & 31) == 0) wparts[threadIdx.x >> 5] = __popc(opens);
        __syncthreads();
        part = (uint32_t)pd.part_cnt[blockIdx.x] + __popc(opens & ka_lanemask_lt());
        for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) part += wparts[w];
    }
    const unsigned long long at = d.blockoff[blockIdx.x];   // this CTA's text
    char* dst = d.p.json + at;
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(dst) & 15u);
    char* stage = reinterpret_cast<char*>(ka_jsmem) + mis;
    const bool staged = mis + bt <= KA_JSON_SMEM_BYTES;
    if (i < M) {
        uint32_t g;
        int v;
        bool first, last;
        ka_wave_doc_row<PARTS>(d, pd, i, M, g, v, first, last);
        char* w = (staged ? stage : dst) + loc;
        if constexpr (BACK) {   // part is the number of parts opened before i: with i's own, D at the last row
            if (first) {
                w = ka_put_str(w, KA_BACK_HEAD, KA_BACK_HEAD_LEN);
                d.doc_off[part] = at + loc;
            }
            w = ka_json_back_put(d.p, bk.rep_off, bk.cur, g, w, !first);
            if (last) ka_put_str(w, KA_BACK_TAIL, KA_BACK_TAIL_LEN);
            if (i + 1 == M) d.doc_off[part + (first ? 1u : 0u)] = at + loc + n;
        } else {
            if (first) {
                w = ka_put_str(w, KA_JSON_HEAD, KA_JSON_HEAD_LEN);
                if constexpr (PARTS) {
                    d.doc_off[part] = at + loc;
                    pd.doc_wave[part] = v;
                } else {
                    d.doc_off[v - 1] = at + loc;
                }
            }
            w = ka_json_row_put(d.p, g, w, !first);
            if (last) ka_put_str(w, KA_JSON_TAIL, KA_JSON_TAIL_LEN);
            if (i + 1 == M) {
                if constexpr (PARTS) d.doc_off[total[1]] = at + loc + n;
                else d.doc_off[v] = at + loc + n;
            }
        }
    }
    if (staged) ka_json_store_staged(dst, stage, bt);
}

// The part passes of a size limit, over the grouped positions of d (d.p.rowlen holds c_i, d.blockoff their CTA sums and then
// offsets). Positions i..j-1 of one wave make one part iff S[j] - S[i] <= room = L - 28.
struct KaWaveParts {
    KaWaveDocs d;
    long long room;
    unsigned long long* S;          // [M + 1]
    int32_t* first_pos;             // [W + 1] first position of every wave, M at W
    int32_t* next;                  // [M] J_0
    uint8_t* start;                 // [M] 1 at the wave starts (then, by the mark passes, at every part start)
    unsigned long long* err;        // (row << 32) | its one-record document's bytes (clipped), of the lowest row that exceeds L
    unsigned long long* widest;     // the most rows of a wave
};

// grid ceil(Q / 256), 256 threads. BACK: c'_i and its CTA sums too. CAPS: a_i and its CTA sums too.
template <bool BACK, bool CAPS>
__global__ void __launch_bounds__(256) ka_wave_part_len_kernel(const KaWaveParts pp, const KaWaveBack bk, const KaWaveCaps cp) {
    const KaWaveDocs& d = pp.d;
    const uint32_t M = (uint32_t)*d.n_rows;
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    uint32_t c = 0, cb = 0;
    unsigned long long a = 0;
    if (i < M) {
        uint32_t g;
        int v;
        bool first, last;
        ka_wave_doc_row<false>(d, KaWaveDocParts{}, i, M, g, v, first, last);
        c = ka_json_row_len(d.p, g, true);   // the record and its comma
        d.p.rowlen[i] = c;
        if constexpr (BACK) {
            cb = ka_json_back_len(d.p, bk.rep_off, bk.cur, g, true);
            bk.rowlen[i] = cb;
        }
        if constexpr (CAPS) {   // what ka_wave_sum_kernel adds to replicas_added for the row
            const int nr = cp.nrecv[g];
            a = nr > 0 ? (unsigned long long)nr * (unsigned long long)(cp.weight ? __ldg(cp.weight + g) : 1) : 0ull;
            cp.A[i] = a;
        }
        pp.start[i] = first;
        if (first) pp.first_pos[v - 1] = (int32_t)i;
        if (i + 1 == M) pp.first_pos[v] = (int32_t)M;
    }
    const unsigned long long bytes = ka_cta256_sum(c);
    if (threadIdx.x == 0) d.blockoff[blockIdx.x] = bytes;
    if constexpr (BACK) {
        __syncthreads();   // thread 0 has read the warp sums: the second sum may write them
        const unsigned long long back = ka_cta256_sum(cb);
        if (threadIdx.x == 0) bk.blockoff[blockIdx.x] = back;
    }
    if constexpr (CAPS) {   // its own shared words: no barrier needed before it
        unsigned long long sum;
        ka_cta256_prefix64(a, sum);
        if (threadIdx.x == 0) cp.blockoff[blockIdx.x] = sum;
    }
}

// ONE CTA of 1024: K arrays of CTA sums to their offsets, in place: v and w (K = 2: S and R, or S and A), and x (K = 3: A
// beside S and R).
template <int K>
__global__ void __launch_bounds__(1024) ka_wave_part_scan_kernel(unsigned long long* __restrict__ v, unsigned long long* __restrict__ w,
                                                                 int n, unsigned long long* __restrict__ x) {
    ka_cta_scan(v, v, n, 0ull);
    __syncthreads();   // every thread has read the first scan's total: the second may reset it
    ka_cta_scan(w, w, n, 0ull);
    if constexpr (K == 3) {
        __syncthreads();
        ka_cta_scan(x, x, n, 0ull);
    }
}

// grid ceil(Q / 256), 256 threads: S[i] = the CTA's offset + the in-CTA prefix; the last position also writes S[M]. BACK: R
// likewise. CAPS: A likewise, over the a_i the length pass left in A (each thread reads only its own).
template <bool BACK, bool CAPS>
__global__ void __launch_bounds__(256) ka_wave_part_prefix_kernel(const KaWaveParts pp, const KaWaveBack bk, const KaWaveCaps cp) {
    const uint32_t M = (uint32_t)*pp.d.n_rows;
    if (blockIdx.x * 256u >= M) return;   // CTA-uniform
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    const uint32_t c = i < M ? pp.d.p.rowlen[i] : 0u;
    uint32_t bt;
    const unsigned long long s = pp.d.blockoff[blockIdx.x] + ka_cta256_prefix(c, bt);
    if (i < M) pp.S[i] = s;
    if (i + 1 == M) pp.S[M] = s + c;
    if constexpr (BACK) {
        __syncthreads();   // every thread has read the warp sums
        const uint32_t cb = i < M ? bk.rowlen[i] : 0u;
        const unsigned long long r = bk.blockoff[blockIdx.x] + ka_cta256_prefix(cb, bt);
        if (i < M) bk.R[i] = r;
        if (i + 1 == M) bk.R[M] = r + cb;
    }
    if constexpr (CAPS) {
        const unsigned long long a = i < M ? cp.A[i] : 0ull;
        unsigned long long sum;
        const unsigned long long x = cp.blockoff[blockIdx.x] + ka_cta256_prefix64(a, sum);
        if (i < M) cp.A[i] = x;
        if (i + 1 == M) cp.A[M] = x + a;
    }
}

// CAPS: whether a part opened at a position with A = a0 may end at j (j > that position + 1) within the data cap.
template <bool CAPS>
__device__ __forceinline__ bool ka_wave_part_in(const KaWaveCaps& cp, uint32_t j, unsigned long long a0) {
    if constexpr (CAPS) return cp.A[j] - a0 <= cp.in;
    return true;
}

// grid ceil(Q / 256), 256 threads: J_0[i] = the last j in (i, e] with S[j] - S[i] <= room, e the end of i's wave, and M in
// place of e. A position whose own record does not fit reports its ROW, so the lowest input row wins. BACK: the last j that
// also keeps R[j] - R[i] <= room (both conditions are monotone in j); a record that does not fit on either side reports the
// longer one-record document. CAPS: j also at most i + Lr, and A[j] - A[i] <= Lx for j > i + 1 (monotone too: a >= 0).
template <bool BACK, bool CAPS>
__global__ void __launch_bounds__(256) ka_wave_part_next_kernel(const KaWaveParts pp, const KaWaveBack bk, const KaWaveCaps cp) {
    const uint32_t M = (uint32_t)*pp.d.n_rows;
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    if (i >= M) return;
    const uint32_t g = (uint32_t)pp.d.perm[i];
    const int v = pp.d.wave[g];
    const uint32_t e = (uint32_t)pp.first_pos[v];
    if (pp.start[i]) atomicMax(pp.widest, (unsigned long long)(e - i));
    const long long lim = (long long)pp.S[i] + pp.room;
    if constexpr (BACK) {
        const long long lim_r = (long long)bk.R[i] + pp.room;
        if ((long long)pp.S[i + 1] > lim || (long long)bk.R[i + 1] > lim_r) {
            const unsigned long long rec = max(pp.S[i + 1] - pp.S[i], bk.R[i + 1] - bk.R[i]);
            atomicMin(pp.err, (unsigned long long)g << 32 | min(28ull + rec, 0xFFFFFFFFull));
            return;
        }
        uint32_t lo = i + 1, hi = e;   // S[lo] <= lim and R[lo] <= lim_r
        unsigned long long a0 = 0;   // CAPS: the search ends at i + Lr, and a run holds at most Lx above A[i]
        if constexpr (CAPS) hi = (uint32_t)min((unsigned long long)e, (unsigned long long)i + cp.rows), a0 = cp.A[i];
        while (lo < hi) {
            const uint32_t mid = (lo + hi + 1) >> 1;
            if ((long long)pp.S[mid] <= lim && (long long)bk.R[mid] <= lim_r && ka_wave_part_in<CAPS>(cp, mid, a0)) lo = mid; else hi = mid - 1;
        }
        pp.next[i] = (int32_t)(lo == e ? M : lo);
        return;
    }
    if ((long long)pp.S[i + 1] > lim) {
        const unsigned long long bytes = min(28ull + (pp.S[i + 1] - pp.S[i]), 0xFFFFFFFFull);
        atomicMin(pp.err, (unsigned long long)g << 32 | bytes);
        return;
    }
    uint32_t lo = i + 1, hi = e;   // S[lo] <= lim
    unsigned long long a0 = 0;   // CAPS: the search ends at i + Lr, and a run holds at most Lx above A[i]
    if constexpr (CAPS) hi = (uint32_t)min((unsigned long long)e, (unsigned long long)i + cp.rows), a0 = cp.A[i];
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if ((long long)pp.S[mid] <= lim && (!CAPS || ka_wave_part_in<CAPS>(cp, mid, a0))) lo = mid; else hi = mid - 1;
    }
    pp.next[i] = (int32_t)(lo == e ? M : lo);
}

// grid ceil(M / 256), 256 threads: J_k from J_{k-1}; M stays M.
__global__ void __launch_bounds__(256) ka_wave_part_jump_kernel(const int32_t* __restrict__ J, int32_t* __restrict__ J2, uint32_t M) {
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    if (i >= M) return;
    const int32_t j = J[i];
    J2[i] = (uint32_t)j == M ? j : J[j];
}

// grid ceil(M / 256), 256 threads: one level of the top-down marking. A start read here may have been set in this same pass;
// its image is a start all the same.
__global__ void __launch_bounds__(256) ka_wave_part_mark_kernel(const int32_t* __restrict__ J, uint8_t* start, uint32_t M) {
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    if (i >= M || !start[i]) return;
    const int32_t j = J[i];
    if ((uint32_t)j != M) start[j] = 1;
}
