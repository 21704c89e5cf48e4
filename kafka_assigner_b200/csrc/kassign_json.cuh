// kassign_json.cuh — the reassignment JSON of KafkaAssignmentGenerator.printLeastDisruptiveReassignment (KAG:169-186) built
// on the device from the solved rows, so that only TEXT crosses PCIe and it can stream out fragment by fragment while later
// topic blocks are still in the leader-order chains. Rows are those of a dense run (P partitions 0..P-1 per topic) or of a
// ragged one (part_off / part_id, as ka_solve takes them).
//
//   {"partitions":[{"partition":P,"replicas":[a,b,c],"topic":"name"},...],"version":1}
//
// org.json 20131018 prints object keys in java.util.HashMap iteration order (SURVEY.md §3.4): "partitions" before "version",
// "partition" / "replicas" / "topic" inside a record — predicted, unverified without a JVM; the order lives only in
// ka_json_row_len / ka_json_row_put below (and in kassign_host.hpp::newAssignmentJson for the host emitter).
// Topic names must not need JSON escaping (Kafka topic names are [a-zA-Z0-9._-]); the host checks before choosing this path.
#pragma once
#include "kassign_common.cuh"

struct KaJsonParams {
    uint32_t Q;                 // rows of this fragment
    uint32_t row0;              // index of the fragment's first row in the whole run (row 0 has no leading comma)
    int P;                      // dense shape: partition id = row % P, topic = topic0 + row / P
    int topic0;
    int T;                      // ragged shape (part_off != null): topics of the run
    const int64_t* part_off;    // [T+1] rows of topic t are part_off[t] .. part_off[t+1]-1 (run-wide row indices)
    const int32_t* part_id;     // [rows of the run] partition ids; null = the ordinal inside the topic
    const int64_t* name_off;    // [T+1] byte offsets into names
    const char* names;          // concatenated topic names (UTF-8, no escapes needed)
    const int32_t* out;         // [Q][S] broker ids, leader first
    const int32_t* out_len;     // [Q]
    int S;
    uint32_t* rowlen;           // [Q] scratch
    uint32_t* blocksum;         // [ceil(Q / 256)] scratch
    unsigned long long* total;  // device scalar: bytes written so far (header included); advanced by this fragment
    unsigned long long* frag;   // [2] out: {first byte, byte count} of this fragment (the header / trailer included)
    char* json;
    unsigned long long cap;     // bytes of `json`: a fragment that would end beyond it is measured but NOT written
    int first, last;            // write the header before / the trailer after this fragment
};

// The documents of a segmented pass (SEG = true): the rows of a fleet of K clusters, one document per cluster. Row g belongs
// to the cluster k with row0[k] <= g < row0[k + 1]; cluster k is live when it is a batch member whose run reported no failure.
struct KaJsonSegs {
    int K;
    const int64_t* row0;        // [K+1] first row of every cluster (run-wide), row0[K] = rows of the run
    const int32_t* member;      // [K] batch member of cluster k, -1 = left out of the run
    const unsigned* flags;      // [members] lowest failing topic of every member, 0xFFFFFFFF = none
    unsigned long long* bytes;  // [K] text bytes of cluster k's rows (zeroed by the host, summed by the length pass)
    unsigned long long* doc_off;  // [K+1] out: cluster k's document is json[doc_off[k] .. doc_off[k+1]) (empty when dead)
    uint32_t* shift;            // [K] out: bytes of headers / trailers in front of cluster k's rows
};

#define KA_JSON_HEAD "{\"partitions\":["
#define KA_JSON_TAIL "],\"version\":1}"
#define KA_JSON_HEAD_LEN 15
#define KA_JSON_TAIL_LEN 14
#define KA_JSON_MAX_SEGS 128   // clusters of one segmented pass (the batched solves' member limit)

__device__ __forceinline__ uint32_t ka_ndigits(int32_t v) {  // characters of Integer.toString(v)
    uint32_t u = v < 0 ? 0u - (uint32_t)v : (uint32_t)v, n = v < 0 ? 2u : 1u;
    while (u >= 10u) { u /= 10u; ++n; }
    return n;
}
__device__ __forceinline__ char* ka_put_int(char* p, int32_t v) {
    char tmp[11];
    uint32_t u = v < 0 ? 0u - (uint32_t)v : (uint32_t)v;
    int n = 0;
    do { tmp[n++] = (char)('0' + u % 10u); u /= 10u; } while (u);
    if (v < 0) *p++ = '-';
    while (n) *p++ = tmp[--n];
    return p;
}
__device__ __forceinline__ char* ka_put_str(char* p, const char* s, int n) {
    for (int i = 0; i < n; ++i) p[i] = s[i];
    return p + n;
}

// Topic and partition id of row q of the fragment.
__device__ __forceinline__ void ka_json_row_key(const KaJsonParams& p, uint32_t q, int& t, int& part) {
    if (p.part_off) {
        const int64_t g = (int64_t)p.row0 + q;
        int lo = 0, hi = p.T;  // part_off[lo] <= g < part_off[hi]; a topic without partitions never satisfies both
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (p.part_off[mid] <= g) lo = mid; else hi = mid;
        }
        t = lo;
        part = p.part_id ? p.part_id[g] : (int)(g - p.part_off[lo]);
    } else {
        t = p.topic0 + (int)(q / (uint32_t)p.P);
        part = (int)(q % (uint32_t)p.P);
    }
}

// Text of row q of the fragment, with a leading comma when `comma`: every row but the first of its document has one.
__device__ __forceinline__ uint32_t ka_json_row_len(const KaJsonParams& p, uint32_t q, bool comma) {
    int t, part;
    ka_json_row_key(p, q, t, part);
    const int len = p.out_len[q];
    uint32_t n = (comma ? 1u : 0u) + 13u + ka_ndigits(part) + 13u + 11u + (uint32_t)(p.name_off[t + 1] - p.name_off[t]) + 2u;
    for (int i = 0; i < len; ++i) n += ka_ndigits(p.out[(size_t)q * p.S + i]) + (i ? 1u : 0u);
    return n;
}
// Writes that text at w; returns its end.
__device__ __forceinline__ char* ka_json_row_put(const KaJsonParams& p, uint32_t q, char* w, bool comma) {
    int t, part;
    ka_json_row_key(p, q, t, part);
    const int len = p.out_len[q];
    if (comma) *w++ = ',';
    w = ka_put_str(w, "{\"partition\":", 13);
    w = ka_put_int(w, part);
    w = ka_put_str(w, ",\"replicas\":[", 13);
    for (int i = 0; i < len; ++i) {
        if (i) *w++ = ',';
        w = ka_put_int(w, p.out[(size_t)q * p.S + i]);
    }
    w = ka_put_str(w, "],\"topic\":\"", 11);
    w = ka_put_str(w, p.names + p.name_off[t], (int)(p.name_off[t + 1] - p.name_off[t]));
    return ka_put_str(w, "\"}", 2);
}

// The rollback record of row q: the row's CURRENT list cur[rep_off[g] .. rep_off[g + 1]) (g the run-wide row) as given, in the
// key order of Kafka 0.10's ZkUtils.formatAsReassignmentJson, which prints the "CURRENT ASSIGNMENT" (KAG:103-111):
//   {"topic":"name","partition":P,"replicas":[a,b,c]}
// 39 bytes + name + partition digits + list, as the record of ka_json_row_len: only the list differs. Its document frame is
// {"version":1,"partitions":[ ... ]}, 29 bytes like the other.
#define KA_BACK_HEAD "{\"version\":1,\"partitions\":["
#define KA_BACK_TAIL "]}"
#define KA_BACK_HEAD_LEN 27
#define KA_BACK_TAIL_LEN 2

__device__ __forceinline__ uint32_t ka_json_back_len(const KaJsonParams& p, const int64_t* rep_off, const int32_t* cur, uint32_t q,
                                                     bool comma) {
    int t, part;
    ka_json_row_key(p, q, t, part);
    const int64_t g = (int64_t)p.row0 + q, a = rep_off[g], b = rep_off[g + 1];
    uint32_t n = (comma ? 1u : 0u) + 10u + (uint32_t)(p.name_off[t + 1] - p.name_off[t]) + 14u + ka_ndigits(part) + 13u + 2u;
    for (int64_t i = a; i < b; ++i) n += ka_ndigits(cur[i]) + (i > a ? 1u : 0u);
    return n;
}
__device__ __forceinline__ char* ka_json_back_put(const KaJsonParams& p, const int64_t* rep_off, const int32_t* cur, uint32_t q,
                                                  char* w, bool comma) {
    int t, part;
    ka_json_row_key(p, q, t, part);
    const int64_t g = (int64_t)p.row0 + q, a = rep_off[g], b = rep_off[g + 1];
    if (comma) *w++ = ',';
    w = ka_put_str(w, "{\"topic\":\"", 10);
    w = ka_put_str(w, p.names + p.name_off[t], (int)(p.name_off[t + 1] - p.name_off[t]));
    w = ka_put_str(w, "\",\"partition\":", 14);
    w = ka_put_int(w, part);
    w = ka_put_str(w, ",\"replicas\":[", 13);
    for (int64_t i = a; i < b; ++i) {
        if (i > a) *w++ = ',';
        w = ka_put_int(w, cur[i]);
    }
    return ka_put_str(w, "]}", 2);
}

// The row texts of a CTA of 256 threads, n bytes per thread. ka_cta256_sum: the CTA's bytes, in thread 0. ka_cta256_prefix:
// this thread's offset in the CTA's text, and (total) the CTA's bytes, in every thread.
__device__ __forceinline__ unsigned long long ka_cta256_sum(uint32_t n) {
    __shared__ uint32_t wsum[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(KA_FULL, n, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = n;
    __syncthreads();
    unsigned long long s = 0;
    if (threadIdx.x == 0)
        for (int i = 0; i < 8; ++i) s += wsum[i];
    return s;
}
__device__ __forceinline__ uint32_t ka_cta256_prefix(uint32_t n, uint32_t& total) {
    __shared__ uint32_t wsum[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(KA_FULL, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    uint32_t woff = 0;
    total = 0;
    for (int i = 0; i < 8; ++i) { if (i < warp) woff += wsum[i]; total += wsum[i]; }
    return woff + x - n;
}

// The write passes assemble a CTA's text in shared memory (KA_JSON_SMEM_BYTES, + 16 for the phase) at the same 16-byte phase
// as its destination, then store it with coalesced 16-byte stores; a CTA whose text does not fit (very long topic names)
// writes straight to global memory instead.
#define KA_JSON_SMEM_BYTES (64 * 1024)

// Every thread of a CTA of 256, once each has written its row into stage: the bt bytes at stage to dst, as the bytes up to
// dst's first 16-byte boundary, a uint4 body, then the tail bytes.
__device__ __forceinline__ void ka_json_store_staged(char* dst, const char* stage, uint32_t bt) {
    __syncthreads();
    const uint32_t head = min(bt, (0u - (uint32_t)reinterpret_cast<uintptr_t>(dst)) & 15u);
    for (uint32_t i = threadIdx.x; i < head; i += 256) dst[i] = stage[i];
    const uint32_t body = (bt - head) >> 4;
    const uint4* s4 = reinterpret_cast<const uint4*>(stage + head);
    uint4* d4 = reinterpret_cast<uint4*>(dst + head);
    for (uint32_t i = threadIdx.x; i < body; i += 256) d4[i] = s4[i];
    for (uint32_t i = head + (body << 4) + threadIdx.x; i < bt; i += 256) dst[i] = stage[i];
}

// Segmented passes: the clusters' first rows, and (live != null) whether each cluster is live, in shared memory.
__device__ __forceinline__ void ka_json_stage_segs(const KaJsonSegs& sg, int64_t* row0, int* live) {
    for (int k = threadIdx.x; k <= sg.K; k += blockDim.x) {
        row0[k] = sg.row0[k];
        if (live && k < sg.K) live[k] = sg.member[k] >= 0 && sg.flags[sg.member[k]] == 0xFFFFFFFFu;
    }
}
// The cluster of run-wide row g < seg_row0[K] (a cluster without rows never satisfies row0[k] <= g < row0[k + 1]).
__device__ __forceinline__ int ka_json_seg_of(const int64_t* row0, int K, int64_t g) {
    int lo = 0, hi = K;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (row0[mid] <= g) lo = mid; else hi = mid;
    }
    return lo;
}

// pass 1: text length of every row + per-block sums. The first row of the run has no leading comma; SEG: the first row of
// every cluster has none, the rows of a dead cluster are empty, and every cluster's bytes are summed into sg.bytes (one atomic
// per warp and cluster).
template <bool SEG>
__global__ void __launch_bounds__(256) ka_json_len_kernel(const KaJsonParams p, const KaJsonSegs sg) {
    const uint32_t q = blockIdx.x * 256u + threadIdx.x;
    uint32_t n;
    if constexpr (SEG) {
        __shared__ int64_t row0[KA_JSON_MAX_SEGS + 1];
        __shared__ int live[KA_JSON_MAX_SEGS];
        ka_json_stage_segs(sg, row0, live);
        __syncthreads();
        const int64_t g = (int64_t)p.row0 + q;
        const int k = q < p.Q ? ka_json_seg_of(row0, sg.K, g) : -1;
        n = k >= 0 && live[k] ? ka_json_row_len(p, q, g != row0[k]) : 0u;
        const unsigned grp = __match_any_sync(KA_FULL, k);
        const unsigned sum = __reduce_add_sync(grp, n);
        if (k >= 0 && sum > 0 && (int)(threadIdx.x & 31) == __ffs(grp) - 1) atomicAdd(sg.bytes + k, (unsigned long long)sum);
    } else {
        n = q < p.Q ? ka_json_row_len(p, q, p.row0 + q > 0) : 0u;
    }
    if (q < p.Q) p.rowlen[q] = n;
    const unsigned long long bytes = ka_cta256_sum(n);
    if (threadIdx.x == 0) p.blocksum[blockIdx.x] = (uint32_t)bytes;
}

// pass 2 (one CTA): exclusive scan of the block sums, relative to the fragment start (a fragment is < 4 GiB), after the
// header's reserve; the fragment, with its trailer's, is placed after the bytes written so far
__global__ void __launch_bounds__(1024) ka_json_scan_kernel(const KaJsonParams p, int nblocks) {
    const unsigned long long base = *p.total;   // loaded ahead of the scan, off the path to the stores below
    const unsigned long long bytes =
        ka_cta_scan(p.blocksum, p.blocksum, nblocks, (unsigned long long)(p.first ? KA_JSON_HEAD_LEN : 0)) + (p.last ? KA_JSON_TAIL_LEN : 0);
    if (threadIdx.x == 0) {
        p.frag[0] = base;
        p.frag[1] = bytes;
        *p.total = base + bytes;
    }
}

// Segmented passes, after the last fragment's scan (one CTA of KA_JSON_MAX_SEGS threads): the document table. Rows are in
// cluster order and a dead cluster's rows are empty, so the rows of cluster k start at sum_{j<k} sg.bytes[j] of the row
// text, and its document 29 bytes per live cluster before it later. Writes doc_off, shift and every live cluster's header
// and trailer (the whole document of a live cluster without rows); no text when it would end beyond p.cap.
__global__ void __launch_bounds__(KA_JSON_MAX_SEGS) ka_json_docs_kernel(const KaJsonParams p, const KaJsonSegs sg) {
    __shared__ int64_t row0[KA_JSON_MAX_SEGS + 1];
    __shared__ int live[KA_JSON_MAX_SEGS];
    __shared__ unsigned long long off[KA_JSON_MAX_SEGS + 1];
    ka_json_stage_segs(sg, row0, live);
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long o = 0;
        uint32_t before = 0;
        for (int k = 0; k < sg.K; ++k) {
            off[k] = o;
            sg.shift[k] = KA_JSON_HEAD_LEN + (KA_JSON_HEAD_LEN + KA_JSON_TAIL_LEN) * before;
            if (live[k]) {
                o += KA_JSON_HEAD_LEN + KA_JSON_TAIL_LEN + sg.bytes[k];
                ++before;
            }
        }
        off[sg.K] = o;
    }
    __syncthreads();
    for (int k = threadIdx.x; k <= sg.K; k += blockDim.x) {
        sg.doc_off[k] = off[k];
        if (k < sg.K && live[k] && off[sg.K] <= p.cap) {
            ka_put_str(p.json + off[k], KA_JSON_HEAD, KA_JSON_HEAD_LEN);
            ka_put_str(p.json + off[k + 1] - KA_JSON_TAIL_LEN, KA_JSON_TAIL, KA_JSON_TAIL_LEN);
        }
    }
}

// pass 3: every row writes its text at its final position, the 256 rows of a block through the shared-memory stage.
// SEG: a row's position moves by its cluster's shift, so a block whose rows span documents (the shift differs at its ends)
// writes straight to global memory.
template <bool SEG>
__global__ void __launch_bounds__(256) ka_json_write_kernel(const KaJsonParams p, const KaJsonSegs sg) {
    extern __shared__ __align__(16) unsigned char ka_jsmem[];
    if (SEG ? sg.doc_off[sg.K] > p.cap : p.frag[0] + p.frag[1] > p.cap) return;   // caller's buffer too small (uniform)
    const uint32_t q = blockIdx.x * 256u + threadIdx.x;
    const uint32_t n = q < p.Q ? p.rowlen[q] : 0u;
    uint32_t bt;
    const uint32_t loc = ka_cta256_prefix(n, bt);               // my row inside the block's text
    uint32_t shift = 0, bshift = 0;   // position shift of my row and of the block's first row
    bool staged = true, comma = p.row0 + q > 0;
    if constexpr (SEG) {
        __shared__ int64_t row0[KA_JSON_MAX_SEGS + 1];
        ka_json_stage_segs(sg, row0, nullptr);
        __syncthreads();
        const uint32_t q0 = blockIdx.x * 256u, q1 = min(p.Q, q0 + 256u) - 1;
        bshift = sg.shift[ka_json_seg_of(row0, sg.K, (int64_t)p.row0 + q0)];
        staged = bshift == sg.shift[ka_json_seg_of(row0, sg.K, (int64_t)p.row0 + q1)];
        if (q < p.Q) {
            const int64_t g = (int64_t)p.row0 + q;
            const int k = ka_json_seg_of(row0, sg.K, g);
            shift = sg.shift[k];
            comma = g != row0[k];
        }
    }
    char* frag = p.json + p.frag[0];
    char* dst = frag + p.blocksum[blockIdx.x] + bshift;        // this block's text
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(dst) & 15u);
    // SEG: a dead cluster's rows are empty and never read
    if (staged && mis + bt <= KA_JSON_SMEM_BYTES) {
        char* stage = reinterpret_cast<char*>(ka_jsmem) + mis;
        if (SEG ? n > 0 : q < p.Q) ka_json_row_put(p, q, stage + loc, comma);
        ka_json_store_staged(dst, stage, bt);
    } else if (SEG ? n > 0 : q < p.Q) {
        ka_json_row_put(p, q, dst + loc + (shift - bshift), comma);
    }
    if constexpr (!SEG) {   // a segmented pass's headers and trailers come from ka_json_docs_kernel
        if (q == 0 && p.first) ka_put_str(frag, KA_JSON_HEAD, KA_JSON_HEAD_LEN);
        if (q == 0 && p.last) ka_put_str(frag + p.frag[1] - KA_JSON_TAIL_LEN, KA_JSON_TAIL, KA_JSON_TAIL_LEN);
    }
}
