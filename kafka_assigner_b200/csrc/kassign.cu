// kassign.cu — C ABI (include/kassign.h) over the sm_90a kernels in kassign_stage.cuh / kassign_order.cuh / kassign_json.cuh.
//
// Reference boundary: KafkaTopicAssigner.generateAssignment (KafkaTopicAssigner.java:42-72) batched over
// the topic loop of KafkaAssignmentGenerator.java:172-184. No CPU fallback exists in this library.
#include "kassign_stage.cuh"
#include "kassign_order.cuh"
#include "kassign_json.cuh"
#include "kassign_score.cuh"
#include "kassign_waves.cuh"
#include "kassign_waves_json.cuh"
#include "kassign_usage.cuh"

#include <algorithm>
#include <array>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <new>
#include <optional>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/kassign.h"

namespace {

constexpr int KA_SM_COUNT_FALLBACK = 132;   // H100 SXM
constexpr size_t KA_SMEM_BUDGET = 200 * 1024;   // per-CTA dynamic smem we allow ourselves (of 227 KB)
constexpr uint32_t KA_LUT_SMEM_MAX_RANGE = 32768;
constexpr uint32_t KA_LUT_GLOBAL_MAX_RANGE = 1u << 25;

// A device allocation that only grows, freed with its owner (ka_ctx_destroy deletes the ctx with its device current).
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        release();
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

constexpr int KA_MAX_BLOCKS = 8;          // topic blocks of a pipelined solve
constexpr int KA_MAX_CHAIN_BLOCKS = 16;   // slot-chain sub-blocks per staged block
constexpr int KA_MAX_CHAIN_EVENTS = KA_MAX_BLOCKS * KA_MAX_CHAIN_BLOCKS;   // chain sub-blocks per solve
// JSON fragments of one solve: one per chain sub-block of a dense solve; a ragged solve (one block, one sub-block) cuts its
// rows into fragments of KA_JSON_FRAG_ROWS rows (more per fragment only beyond KA_MAX_JSON_FRAGS of them), so that the text
// streams out while later fragments are still being built and every fragment stays far below the 4 GiB of its 32-bit offsets.
constexpr int KA_MAX_JSON_FRAGS = 256;
constexpr int KA_MAX_CANDIDATES = 128;    // candidate broker tables of one batched solve
static_assert(KA_MAX_CANDIDATES <= KA_JSON_MAX_SEGS, "a fleet's documents are built in one segmented JSON pass");
constexpr int64_t KA_JSON_FRAG_ROWS = 1 << 18;

struct HostPinned {
    int err_topic;
    int spin_flag;
    int4 tstatus;
};

struct Plan {
    // kernel A
    int a_blob_bytes;                               // shared memory for the broker blob (the largest of a batched solve)
    int a_warps, a_load_bytes, a_slab_bytes, a_cnt_bytes, a_load_kind;  // kind 0=u8 1=u16
    int a_levels;                                   // 1: some topic may hold a broker twice -> conflict levels + tables
    int lv_owner_bytes, lv_last_bytes, lv_p_bytes;  // per-warp scratch of the level pass
    size_t a_smem;
    // leader order
    int rec_kind, rec_bytes;  // 3: 16 B records (rows <= 3), 4 / 8: 32 B records (rows of 4 / 5..8)
    int b_gctr;               // counters stay in global memory (table too large for shared memory)
    int b_ring_log2;          // log2(records per TMA ring stage)
    int b_threads;
    size_t b_smem;
};

// One contiguous block of topics of a dense or ragged problem, with every device pointer already offset to the block.
struct StageDesc {
    int topic_base = 0, T = 0;
    int64_t Q = 0;                  // partitions in the block
    const int32_t* d_hash = nullptr;
    const int64_t* d_part_off = nullptr;  // ragged only (block == whole problem)
    const int64_t* d_rep_off = nullptr;
    int P = 0, RF = 0;
    const int32_t* d_cur = nullptr;
    int desired_rf = -1, S = 1, Pmax = 0;
    int64_t capmax = 0;
    int64_t q0 = 0;                 // first partition row of the block inside the ctx scratch arrays
    int blk = 0;                    // ordinal of the block inside a pipelined solve (its level tables: loff at topic_base + blk)
    Plan pl;
};

// Records, level tables and status of one run of kernel A and the chains.
struct RunScratch {
    DevBuf rec, perm, ntl, lend, loff, lvl_end, tstatus, flags;
    // rec_bytes of records, q partitions and T topics (nloff chunk-table offsets: the level tables only with levels), nflags
    // status words.
    cudaError_t reserve(size_t rec_bytes, size_t q, size_t T, size_t nloff, bool levels, size_t nflags) {
        const struct { DevBuf* b; size_t bytes; } want[] = {
            {&rec, rec_bytes}, {&perm, levels ? q * 2 : 0}, {&lend, levels ? q * 4 : 0}, {&lvl_end, levels ? q * 4 : 0},
            {&ntl, levels ? T * 4 : 0}, {&loff, levels ? nloff * 4 : 0}, {&tstatus, T * sizeof(int4)}, {&flags, nflags * 4},
        };
        for (const auto& w : want)
            if (cudaError_t e = w.b->reserve(w.bytes)) return e;
        return cudaSuccess;
    }
};

}  // namespace

struct ka_ctx {
    int device = 0;
    int sm_count = KA_SM_COUNT_FALLBACK;
    cudaStream_t stream = nullptr;  // used by the host-buffer entry points
    cudaStream_t aux = nullptr;     // stage of the pipelined (super-chunk) solve
    cudaStream_t sb1 = nullptr;     // slot-0 chains (the slot-1 chains + emit run on the caller's stream)
    cudaStream_t sj = nullptr;      // device JSON emission, streamed copy-out
    std::array<cudaStream_t*, 4> streams() { return {&stream, &aux, &sb1, &sj}; }
    // broker table: the kernels' view of it (in d_blob, d_glut, d_broker_id; N = 0 before ka_ctx_set_brokers) and its ids
    KaBrokers br{};
    std::vector<int32_t> broker_id;
    DevBuf d_blob, d_glut, d_broker_id, d_ctr8;
    // counters of brokers not in the current table (Context.counter is keyed by broker id)
    std::unordered_map<int32_t, std::vector<int32_t>> parked;
    int64_t launches = 0;
    // scratch
    DevBuf d_hash, d_part_off, d_rep_off, d_cur, d_out, d_out_len;
    RunScratch run;   // kernel A and the chains of a single solve (and of a staged block)
    DevBuf d_json, d_names, d_name_off, d_part_id, d_json_rowlen, d_json_blocksum, d_json_state;
    DevBuf d_json_seg;   // the cluster table of ka_solve_clusters_json and ka_score_clusters (the arrays of KaJsonSegs)
    // scratch of the batched solves, apart from the single solve's: descriptors + broker tables, counters, and the run
    DevBuf d_batch_tab, d_batch_ctr;
    RunScratch batch_run;
    // scratch of ka_score_candidates / ka_score_clusters: row weights, and the score passes' arrays (score_batch)
    DevBuf d_score_w, d_score;
    // scratch of ka_plan_waves (its rows: upload_wave_rows): every row's wave, the plan passes' arrays (wave_plan_device), the
    // chain's per-row words when they leave shared memory and the summaries
    DevBuf d_wv_wave, d_wv_plan, d_wv_state, d_wv_sum;
    // scratch of the sender budget (ka_plan_waves_send and its JSON form): the send table, the sender bucket log and the sender
    // summaries (the per-sender words share d_wv_state)
    DevBuf d_wv_send, d_wv_slog, d_wv_ssum;
    // the wave rule of every plan call (ka_ctx_set_wave_rule) and, under KA_WAVE_FIRST_FIT, the load table [N + ns][Wb] (the
    // counts and the chain's per-row words share d_wv_state)
    int32_t wave_rule = KA_WAVE_GREEDY;
    DevBuf d_wv_fit;
    // scratch of ka_plan_waves_json, beside the plan's and the JSON passes' (d_part_off, d_part_id, d_names, d_name_off, d_json,
    // d_json_rowlen, d_json_blocksum as 64-bit offsets): the radix passes' arrays (enq_wave_group), and the text total followed
    // by doc_off [W + 1] (with a size limit: the total, D, then doc_off [D + 1])
    DevBuf d_wv_sort, d_wv_doc;
    // scratch of a size limit (ka_plan_waves_json_parts): the part passes' arrays (enq_wave_parts) and the jump tables J_k, k > 0
    DevBuf d_wv_part, d_wv_jump;
    // the part caps of every _parts call (ka_ctx_set_part_caps): the most rows and the most data of one part, 0 = no cap
    int64_t part_rows = 0, part_in = 0;
    // scratch of the rollback documents (ka_plan_waves_json_parts_rollback): the text, then the rollback side's arrays
    DevBuf d_wv_back, d_wv_bscr;
    // scratch of ka_wave_broker_usage (its rows: upload_wave_rows): the usage passes' arrays
    DevBuf d_usage;
    HostPinned* h_pin = nullptr;
    unsigned long long* h_frag = nullptr;  // pinned [KA_MAX_JSON_FRAGS][2]: {first byte, bytes} of every JSON fragment
    // timing events (recorded only with timing on)
    cudaEvent_t ev[6] = {};                                // solve: start, inputs in, kernel A done, stage done, chains done, end
    cudaEvent_t ev_pipe[KA_MAX_BLOCKS][5] = {};            // pipelined block: stage start, kernel A done, stage done, chains start / done
    cudaEvent_t ev_chain[KA_MAX_BLOCKS][4] = {};           // chains of a block: slot-0 chains start / done (a solve: [0] only), slot-1 chains + emits start / done
    // cross-stream events: ev_b1 / ev_b2 = slot-0 / slot-1 chain of a sub-block done, ev_emit_done = a block's emits done
    cudaEvent_t ev_in = nullptr, ev_stage[KA_MAX_BLOCKS] = {}, ev_chain_in = nullptr, ev_b1[KA_MAX_CHAIN_EVENTS] = {};
    cudaEvent_t ev_b2[KA_MAX_CHAIN_EVENTS] = {}, ev_emit_done = nullptr;
    cudaEvent_t ev_json_in[KA_MAX_JSON_FRAGS] = {}, ev_json_scan[KA_MAX_JSON_FRAGS] = {}, ev_out_done = nullptr;
    // end of the last asynchronous call that leaves no status pending (stage, slot chain, counter import / export), recorded on
    // its stream; the next host call waits for it (enter_host)
    cudaEvent_t ev_tail = nullptr;
    bool tail_pending = false;
    // timing of the last solve
    bool timing = false;
    float last_ms[8] = {};
    bool ev_valid = false;
    int last_stages = 1;
    int chain_used = 0;                    // ev_chain rows recorded (one per block of a solve)
    bool slot_timed[2] = {false, false};   // ka_order_slot_device recorded ev_chain[slot][0..1]
    int32_t order_plan[8] = {};            // ka_ctx_last_order_plan: the leader-order chains of the last solve call
    int32_t stage_plan[8] = {};            // ka_ctx_last_stage_plan: kernel A of the last solve call
    // staged problem (between the context-free stage and the leader-order stage)
    bool staged = false;
    StageDesc staged_block;
    int topic_base = 0;       // ka_ctx_set_topic_base: index of the staged block's first topic in the whole (multi-GPU) run
    // async status
    bool last_was_staged = false;
    cudaStream_t last_stream = nullptr;
    bool pending_status = false;
    ka_status last{};
};

namespace {

#define KA_CUDA(call)                                                                              \
    do {                                                                                           \
        cudaError_t _e = (call);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            std::fprintf(stderr, "[kassign] CUDA error %s at %s:%d: %s\n", cudaGetErrorName(_e), __FILE__, __LINE__, \
                         cudaGetErrorString(_e));                                                  \
            return KA_ERR_CUDA;                                                                    \
        }                                                                                          \
    } while (0)

int set_status(ka_status* st, int code, int topic = -1, int part = -1, int a = 0, int b = 0) {
    if (st) {
        st->code = code;
        st->topic_index = topic;
        st->partition = part;
        st->a = a;
        st->b = b;
    }
    return code;
}

// An internal step failed with rc: report it in *st, unless *st already holds rc with its details (make_plan's limits).
int failed(ka_status* st, int rc) {
    if (st && st->code != rc) set_status(st, rc);
    return rc;
}

inline size_t align16(size_t v) { return (v + 15) & ~size_t(15); }

// The arrays of one scratch, each at a 16-byte boundary, listed once by a function that takes them in order (braced
// initializers evaluate in order, function arguments do not). Run over a Layout without a base, the function sums their bytes
// (layout_bytes); over one at the scratch's memory, a DevBuf's or a host image's, it returns their pointers (place).
struct Layout {
    unsigned char* base = nullptr;
    size_t bytes = 0;
    template <typename T> T* take(size_t n) {
        T* p = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
        bytes += align16(n * sizeof(T));
        return p;
    }
};
template <typename F> size_t layout_bytes(const F& lay) { Layout l; lay(l); return l.bytes; }
template <typename F> auto place(const F& lay, void* base) { Layout l{static_cast<unsigned char*>(base)}; return lay(l); }
// `buf` reserved for the scratch `lay` lists, and the scratch placed there; nullopt when the reserve fails.
template <typename F> auto reserve_layout(DevBuf& buf, const F& lay) -> std::optional<decltype(place(lay, nullptr))> {
    if (buf.reserve(layout_bytes(lay)) != cudaSuccess) return std::nullopt;
    return place(lay, buf.p);
}

// Every event of the ctx, with whether it is timed.
template <typename F>
void for_each_event(ka_ctx* c, F f) {
    const struct { cudaEvent_t* e; size_t n; bool timed; } pools[] = {
        {c->ev, sizeof(c->ev) / sizeof(cudaEvent_t), true},
        {&c->ev_pipe[0][0], sizeof(c->ev_pipe) / sizeof(cudaEvent_t), true},
        {&c->ev_chain[0][0], sizeof(c->ev_chain) / sizeof(cudaEvent_t), true},
        {&c->ev_in, 1, false},
        {c->ev_stage, KA_MAX_BLOCKS, false},
        {&c->ev_chain_in, 1, false},
        {c->ev_b1, KA_MAX_CHAIN_EVENTS, false},
        {c->ev_b2, KA_MAX_CHAIN_EVENTS, false},
        {&c->ev_emit_done, 1, false},
        {c->ev_json_in, KA_MAX_JSON_FRAGS, false},
        {c->ev_json_scan, KA_MAX_JSON_FRAGS, false},
        {&c->ev_out_done, 1, false},
        {&c->ev_tail, 1, false},
    };
    for (const auto& p : pools)
        for (size_t i = 0; i < p.n; ++i) f(p.e[i], p.timed);
}

// download current device counters into ctx->parked keyed by id
int park_counters(ka_ctx* c) {
    if (c->br.N == 0 || !c->d_ctr8.p) return KA_OK;
    std::vector<int32_t> h((size_t)c->br.N * KA_MAX_SLOTS);
    KA_CUDA(cudaMemcpy(h.data(), c->d_ctr8.p, h.size() * 4, cudaMemcpyDeviceToHost));
    for (int i = 0; i < c->br.N; ++i) {
        const int32_t* row = h.data() + (size_t)i * KA_MAX_SLOTS;
        bool nz = false;
        for (int r = 0; r < KA_MAX_SLOTS; ++r) nz |= row[r] != 0;
        if (nz) c->parked[c->broker_id[i]] = std::vector<int32_t>(row, row + KA_MAX_SLOTS);
        else c->parked.erase(c->broker_id[i]);
    }
    return KA_OK;
}

// What ka_ctx_set_brokers refuses in a broker table.
int check_brokers(int N, const int32_t* broker_id, const int32_t* broker_rack) {
    if (N < 0 || (N > 0 && (!broker_id || !broker_rack))) return KA_ERR_BAD_ARG;
    if (N > 65535) return KA_ERR_LIMIT;
    for (int i = 0; i < N; ++i) {
        if (i > 0 && broker_id[i] <= broker_id[i - 1]) return KA_ERR_BAD_ARG;  // strictly ascending
        if (broker_rack[i] < 0 || broker_rack[i] >= 65535) return KA_ERR_BAD_ARG;
    }
    return KA_OK;
}

// The device image of a (checked) broker table: the blob kernel A stages (rack16 || lut16; the LUT part only in
// KA_LUT_SMEM mode) and, in KA_LUT_GLOBAL mode, the id -> index LUT it reads from global memory.
struct BrokerTable {
    int lut_mode = KA_LUT_SMEM, min_id = 0, lut_off = 0;
    uint32_t range = 0;
    std::vector<uint16_t> blob, glut;
    int blob_bytes() const { return (int)(blob.size() * 2); }
    // The kernels' view of this table of N brokers, uploaded to d_blob / d_glut / d_broker_id.
    KaBrokers device(int N, const uint16_t* d_blob, const uint16_t* d_glut, const int32_t* d_broker_id) const {
        return KaBrokers{N, lut_mode, lut_off, blob_bytes(), min_id, range, d_blob, d_glut, d_broker_id};
    }
};

BrokerTable broker_table(int N, const int32_t* broker_id, const int32_t* broker_rack) {
    BrokerTable t;
    t.min_id = N > 0 ? broker_id[0] : 0;
    const uint64_t range64 = N > 0 ? (uint64_t)((int64_t)broker_id[N - 1] - (int64_t)broker_id[0]) + 1 : 0;
    const size_t npad = align16((size_t)std::max(N, 1) * 2) / 2;  // uint16 elements, 16B multiple
    // compact rack ids in order of first appearance (rack identity is all that matters, KAS:90-94)
    std::vector<uint16_t> rackc(std::max(N, 1), 0);
    {
        std::unordered_map<int32_t, int> seen;
        for (int i = 0; i < N; ++i) {
            auto it = seen.find(broker_rack[i]);
            if (it == seen.end()) it = seen.emplace(broker_rack[i], (int)seen.size()).first;
            rackc[i] = (uint16_t)it->second;
        }
    }
    size_t lut_elems = 0;
    if (range64 <= KA_LUT_SMEM_MAX_RANGE) {
        t.lut_mode = KA_LUT_SMEM;
        t.range = (uint32_t)range64;
        lut_elems = align16((size_t)std::max<uint64_t>(range64, 1) * 2) / 2;
    } else if (range64 <= KA_LUT_GLOBAL_MAX_RANGE) {
        t.lut_mode = KA_LUT_GLOBAL;
        t.range = (uint32_t)range64;
        t.glut.assign((size_t)range64, (uint16_t)KA_DEAD);
        for (int i = 0; i < N; ++i) t.glut[(size_t)((int64_t)broker_id[i] - t.min_id)] = (uint16_t)i;
    } else {
        t.lut_mode = KA_LUT_BSEARCH;
        t.range = 0;
    }
    t.lut_off = (int)npad;
    t.blob.assign(npad + lut_elems, (uint16_t)KA_DEAD);
    for (int i = 0; i < N; ++i) {
        t.blob[i] = rackc[i];
        if (t.lut_mode == KA_LUT_SMEM) t.blob[npad + (size_t)((int64_t)broker_id[i] - t.min_id)] = (uint16_t)i;
    }
    return t;
}

constexpr size_t KA_ORDER_SMEM_BUDGET = 226 * 1024;

// N / blob_bytes: the broker table (the largest one of a batched solve).
int make_plan(int N, int blob_bytes, int64_t Q, int S, int Pmax, int64_t capmax, bool ragged, Plan& pl, ka_status* st) {
    if (Q >= (int64_t)1 << 31) return set_status(st, KA_ERR_LIMIT, -1, -1, INT_MAX, 0);
    // ---- kernel A
    // A broker's load never exceeds the capacity. capmax only counts tables that can serve the target RF (dense_capmax,
    // ragged_capmax), so capmax <= Pmax; capacity > 1 turns the level pass on, whose 15-bit cursors need Pmax <= 32767. So
    // a plan that passes the level check below has capmax <= 32767, and 16-bit loads always suffice.
    pl.a_blob_bytes = blob_bytes;
    pl.a_load_kind = capmax <= 255 ? 0 : 1;
    const int lsz = pl.a_load_kind == 0 ? 1 : 2;
    pl.a_load_bytes = (int)align16((size_t)std::max(N, 1) * lsz);
    pl.a_slab_bytes = (int)align16((size_t)std::max(Pmax, 1) * S * 2);
    pl.a_cnt_bytes = (int)align16((size_t)std::max(Pmax, 1));
    // capacity 1 == every broker holds at most one partition of a topic == the topic is a single conflict level
    pl.a_levels = (capmax > 1 || ragged) ? 1 : 0;
    if (pl.a_levels && Pmax > 32767) return set_status(st, KA_ERR_LIMIT, -1, -1, Pmax, N);  // level cursors are 15-bit
    pl.lv_owner_bytes = pl.a_levels ? (int)align16((size_t)std::max(N, 1) * 4) : 0;
    pl.lv_last_bytes = pl.a_levels ? (int)align16((size_t)std::max(N, 1) * 2) : 0;
    pl.lv_p_bytes = pl.a_levels ? (int)align16((size_t)(std::max(Pmax, 1) + 2) * 2) : 0;
    const size_t per_warp = (size_t)pl.a_load_bytes + pl.a_slab_bytes + pl.a_cnt_bytes + pl.lv_owner_bytes + pl.lv_last_bytes +
                            2 * (size_t)pl.lv_p_bytes;
    const size_t shared = 16 + (size_t)blob_bytes;
    if (shared + per_warp > KA_SMEM_BUDGET) return set_status(st, KA_ERR_LIMIT, -1, -1, Pmax, N);
    pl.a_warps = (int)std::min<size_t>(16, (KA_SMEM_BUDGET - shared) / per_warp);
    pl.a_smem = shared + per_warp * pl.a_warps;
    // ---- leader order
    pl.rec_kind = S <= 3 ? 3 : (S == 4 ? 4 : 8);
    pl.rec_bytes = pl.rec_kind == 3 ? 16 : 32;
    const int cw = pl.rec_kind == 8 ? 8 : 4;
    const int max_nt = pl.rec_kind == 3 ? 1024 : (pl.rec_kind == 4 ? 512 : 256);
    // rows <= 3: each slot chain keeps ONE counter column (+ the dummy broker that pads short rows) in shared memory
    const size_t ctr_bytes = pl.rec_kind == 3 ? (size_t)(std::max(N, 1) + 1) * 4 : (size_t)std::max(N, 1) * cw * 4;
    // record ring: KA_RING_STAGES stages of 2^lg records, as large as fits next to the counter table (<= 128 KB)
    const int lg_max = pl.rec_kind == 3 ? 10 : 9, lg_min = 7;
    auto ring_bytes = [&](int l) { return ((size_t)KA_RING_STAGES << l) * pl.rec_bytes + 256; };
    int lg = lg_max;
    pl.b_gctr = 0;
    while (lg > lg_min && ctr_bytes + ring_bytes(lg) > KA_ORDER_SMEM_BUDGET) --lg;
    if (ctr_bytes + ring_bytes(lg) > KA_ORDER_SMEM_BUDGET) {
        pl.b_gctr = 1;  // counter table beyond shared memory: rows stay in global memory (L2)
        lg = lg_max;
    }
    if (const char* e = std::getenv("KA_ORDER_GLOBAL_CTR")) pl.b_gctr = pl.b_gctr || std::atoi(e);
    pl.b_ring_log2 = lg;
    pl.b_smem = ring_bytes(lg) + (pl.b_gctr ? 0 : ctr_bytes);
    // CTA size ~ level width: a level is one pass of the CTA. Capacity 1: level = topic (P wide). Otherwise a level
    // holds each broker at most once, i.e. at most N / S partitions; measured widths are about half of that.
    int64_t width = pl.a_levels ? std::min<int64_t>(Pmax, std::max<int64_t>(1, N / std::max(S, 1) / 2)) : Pmax;
    // a level wider than the CTA is cut into equal chunks (the kernel is issue-bound there: equal halves cost nothing)
    const int64_t cuts = (std::max<int64_t>(width, 1) + max_nt - 1) / max_nt;
    width = (std::max<int64_t>(width, 1) + cuts - 1) / cuts;
    int nt = (int)std::min<int64_t>(max_nt, ((width + 31) / 32) * 32);
    if (const char* e = std::getenv("KA_ORDER_THREADS")) nt = std::atoi(e);
    nt = std::max(32, std::min(max_nt, (nt / 32) * 32));
    nt = std::min(nt, (KA_RING_STAGES - 1) << lg);
    pl.b_threads = nt;
    return KA_OK;
}

// A kernel's dynamic shared-memory cap belongs to the kernel on its device, not to a ka_ctx: every Context of the process
// sets the same attribute, from any host thread. So the cap only ever rises, under one lock: lowering it to one Context's
// size between another Context's raise and its launch would fail that launch. A cap is no reservation; a launch still gets
// the shared memory it asks for, and occupancy follows from that.
cudaError_t allow_smem_of(const void* kernel, size_t bytes) {
    static std::mutex mu;
    static std::map<std::pair<int, const void*>, size_t> cap;   // (device, kernel) -> the cap set so far
    int dev = 0;
    const cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lock(mu);
    size_t& have = cap[{dev, kernel}];
    if (bytes <= have) return cudaSuccess;
    const cudaError_t r = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (r == cudaSuccess) have = bytes;
    return r;
}

template <typename K>
cudaError_t allow_smem(K kernel, size_t bytes) {
    return allow_smem_of((const void*)kernel, bytes);
}

// A whole problem with its inputs on the device: dense (P partitions of RF replicas per topic), or ragged (d_part_off /
// d_rep_off set, with Q and R from the host-side sizing scan; a ragged problem is always one block). Pmax / capmax: the
// largest topic and capacity under the broker table(s) it is solved against (dense: P and dense_capmax). Made by
// dense_shape or ragged_shape; that of a host-buffer solve gets its device pointers from reserve_io.
struct Shape {
    int T = 0, P = 0, RF = 0, desired_rf = -1, S = 1;
    const int32_t* d_hash = nullptr;
    const int32_t* d_cur = nullptr;
    const int64_t* d_part_off = nullptr;
    const int64_t* d_rep_off = nullptr;
    int64_t Q = 0, R = 0;  // partitions, current replicas
    int Pmax = 0;
    int64_t capmax = 0;
};

// The largest capacity (KAS:65-71) of a dense problem of P partitions per topic and target RF rf_t under a table of n
// brokers: 0 when the table cannot serve rf_t, whose every topic then fails with KA_ERR_RF_GT_BROKERS before it loads a
// broker. The dense counterpart of ragged_capmax, which applies the same rule per topic; so capmax <= P.
int64_t dense_capmax(int P, int rf_t, int n) {
    return n > 0 && rf_t <= n ? ((int64_t)P * std::max(rf_t, 0) + n - 1) / n : 0;
}

// A dense problem solved against one table of N brokers, its inputs at d_hash / d_cur.
Shape dense_shape(int T, int P, int RF, int desired_rf, int S, int N, const int32_t* d_hash = nullptr, const int32_t* d_cur = nullptr) {
    Shape sh{T, P, RF, desired_rf, S, d_hash, d_cur};
    sh.Q = (int64_t)T * P;
    sh.R = sh.Q * RF;
    sh.Pmax = P;
    sh.capmax = dense_capmax(P, desired_rf >= 0 ? desired_rf : RF, N);
    return sh;
}

// A ragged problem of Q partitions and R current replicas.
Shape ragged_shape(int T, int64_t Q, int64_t R, int desired_rf, int S, int Pmax = 0, int64_t capmax = 0) {
    Shape sh{T, 0, 0, desired_rf, S};
    sh.Q = Q;
    sh.R = R;
    sh.Pmax = Pmax;
    sh.capmax = capmax;
    return sh;
}

// The planned StageDesc of topics [t0, t1) of a problem, block `blk` of its solve. N / blob_bytes: the broker table (the
// largest one of a batched solve).
int describe_block(const Shape& sh, int t0, int t1, int blk, int N, int blob_bytes, StageDesc& d, ka_status* st) {
    const bool ragged = sh.d_part_off != nullptr;
    d = StageDesc();
    d.topic_base = t0;
    d.T = t1 - t0;
    d.blk = blk;
    d.q0 = (int64_t)t0 * sh.P;
    d.Q = ragged ? sh.Q : (int64_t)d.T * sh.P;
    d.d_hash = sh.d_hash + t0;
    d.d_part_off = sh.d_part_off;
    d.d_rep_off = sh.d_rep_off;
    d.P = sh.P;
    d.RF = sh.RF;
    d.d_cur = sh.d_cur + d.q0 * sh.RF;
    d.desired_rf = sh.desired_rf;
    d.S = sh.S;
    d.Pmax = sh.Pmax;
    d.capmax = sh.capmax;
    return make_plan(N, blob_bytes, d.Q, d.S, d.Pmax, d.capmax, ragged, d.pl, st);
}

// Scratch of a solve of the blocks ds[0..K) (consecutive: the last one ends the problem).
int reserve_scratch(ka_ctx* c, const StageDesc* ds, int K) {
    const StageDesc& e = ds[K - 1];
    const size_t q = (size_t)std::max<int64_t>(e.q0 + e.Q, 1);
    const size_t T = (size_t)std::max(e.topic_base + e.T, 1);
    KA_CUDA(c->run.reserve(q * ds[0].pl.rec_bytes + 256, q, T, T + K + 1, ds[0].pl.a_levels, 16));
    return KA_OK;
}

// The ctx's device copies of the inputs and rows of a host-buffer solve of sh (a dense_shape or, with `ragged`, a
// ragged_shape), and sh pointed at them.
int reserve_io(ka_ctx* c, Shape& sh, bool ragged) {
    KA_CUDA(c->d_hash.reserve((size_t)std::max(sh.T, 1) * 4));
    if (ragged) {
        KA_CUDA(c->d_part_off.reserve((size_t)(sh.T + 1) * 8));
        KA_CUDA(c->d_rep_off.reserve((size_t)(sh.Q + 1) * 8));
    }
    KA_CUDA(c->d_cur.reserve((size_t)std::max<int64_t>(sh.R, 1) * 4));
    KA_CUDA(c->d_out.reserve((size_t)std::max<int64_t>(sh.Q, 1) * sh.S * 4));
    KA_CUDA(c->d_out_len.reserve((size_t)std::max<int64_t>(sh.Q, 1) * 4));
    sh.d_hash = c->d_hash.as<int32_t>();
    sh.d_cur = c->d_cur.as<int32_t>();
    if (ragged) {
        sh.d_part_off = c->d_part_off.as<int64_t>();
        sh.d_rep_off = c->d_rep_off.as<int64_t>();
    }
    return KA_OK;
}

// flags: [0] lowest failing topic (unsigned atomicMin, 0xFFFFFFFF = none)
int reset_flags(ka_ctx* c, cudaStream_t s) {
    c->h_pin->err_topic = -1;
    c->h_pin->spin_flag = -1;
    c->chain_used = 0;
    c->slot_timed[0] = c->slot_timed[1] = false;
    KA_CUDA(cudaMemsetAsync(c->run.flags.p, 0xFF, 2 * sizeof(int), s));
    return KA_OK;
}

// ncand > 0: kernel A of a batched solve over ncand candidate tables (p.cand), grid.y = candidate. *grid_x: the CTAs per
// candidate it launched.
template <typename LoadT, bool LEVELS, int SM, bool CAND>
cudaError_t launch_stage_t(ka_ctx* c, cudaStream_t s, const KaSolveParams& p, const Plan& pl, int T, int ncand, int* grid_x) {
    auto kern = ka_sticky_spread_kernel<LoadT, LEVELS, SM, CAND>;
    const int threads = pl.a_warps * 32;
    cudaError_t e = allow_smem(kern, pl.a_smem);
    if (e != cudaSuccess) return e;
    int occ = 1;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, pl.a_smem);
    if (e != cudaSuccess) return e;
    int grid = (T + pl.a_warps - 1) / pl.a_warps;
    grid = std::min(grid, std::max(1, std::max(1, occ) * c->sm_count / std::max(ncand, 1)));
    *grid_x = grid;
    kern<<<dim3(grid, std::max(ncand, 1)), threads, pl.a_smem, s>>>(p, pl.a_load_bytes, pl.a_slab_bytes, pl.a_cnt_bytes, pl.lv_owner_bytes,
                                                                 pl.lv_last_bytes, pl.lv_p_bytes);
    return cudaGetLastError();
}

template <typename LoadT, bool LEVELS, bool CAND>
cudaError_t launch_stage(ka_ctx* c, cudaStream_t s, const KaSolveParams& p, const Plan& pl, int T, int ncand, int* grid_x) {
    return p.S <= 3 ? launch_stage_t<LoadT, LEVELS, 3, CAND>(c, s, p, pl, T, ncand, grid_x)
                    : launch_stage_t<LoadT, LEVELS, 8, CAND>(c, s, p, pl, T, ncand, grid_x);
}

void reset_plans(ka_ctx* c) {
    for (int32_t& v : c->order_plan) v = 0;
    for (int32_t& v : c->stage_plan) v = 0;
}

// Kernel A in the instantiation the plan asks for. Loads are 1 or 2 bytes (make_plan); a plan without levels has capacity
// <= 1 and so 1-byte loads. lut_mask: bit m is set when one of the launch's broker tables looks ids up in mode m (KA_LUT_*);
// recorded for ka_ctx_last_stage_plan.
template <bool CAND>
int launch_stage_plan(ka_ctx* c, cudaStream_t s, const KaSolveParams& p, const Plan& pl, int T, int ncand, int lut_mask) {
    cudaError_t e;
    int grid_x = 0;
    if (!pl.a_levels) e = launch_stage<uint8_t, false, CAND>(c, s, p, pl, T, ncand, &grid_x);
    else if (pl.a_load_kind == 0) e = launch_stage<uint8_t, true, CAND>(c, s, p, pl, T, ncand, &grid_x);
    else e = launch_stage<uint16_t, true, CAND>(c, s, p, pl, T, ncand, &grid_x);
    KA_CUDA(e);
    c->launches++;
    int32_t* r = c->stage_plan;
    r[0] = pl.a_load_kind == 0 ? 1 : 2;
    r[1] = pl.a_levels;
    r[2] = p.S <= 3 ? 3 : 8;
    r[3] = ncand;
    r[4] = pl.a_warps;
    r[5] = grid_x;
    r[6] = lut_mask;
    r[7]++;
    return KA_OK;
}

// Kernel A's view of the problem of block d (the broker table and the outputs are set by the caller).
KaSolveParams stage_params(const StageDesc& d) {
    KaSolveParams p{};
    p.T = d.T;
    p.topic_base = d.topic_base;
    p.topic_hash = d.d_hash;
    p.part_off = d.d_part_off;
    p.P = d.P;
    p.rep_off = d.d_rep_off;
    p.RF = d.RF;
    p.cur = d.d_cur;
    p.desired_rf = d.desired_rf;
    p.S = d.S;
    p.Pmax = d.Pmax;
    p.blob_space = d.pl.a_blob_bytes;
    p.rec_kind = d.pl.rec_kind;
    p.chunk_w = d.pl.b_threads;
    return p;
}

// Context-free part of a block (shards across GPUs): kernel A (records in schedule order) + the level tables.
// a_done is recorded at the end of kernel A when timing is on; `done` (if given) when the stage is complete. When kernel A
// ends the stage, `done` goes ahead of a_done, so that the chains waiting for it do not also wait for a timed event record,
// which holds its stream for a few µs.
int enq_stage(ka_ctx* c, cudaStream_t s, const StageDesc& d, cudaEvent_t a_done, cudaEvent_t done = nullptr) {
    const Plan& pl = d.pl;
    RunScratch& r = c->run;
    if (d.T > 0) {
        KaSolveParams p = stage_params(d);
        p.br = c->br;
        p.out.rec = r.rec.as<unsigned char>() + (size_t)d.q0 * pl.rec_bytes;
        p.out.perm = pl.a_levels ? r.perm.as<uint16_t>() + d.q0 : nullptr;
        p.out.ntl = pl.a_levels ? r.ntl.as<int32_t>() + d.topic_base : nullptr;
        p.out.lend = pl.a_levels ? r.lend.as<uint32_t>() + d.q0 : nullptr;
        p.out.tstatus = r.tstatus.as<int4>();
        p.out.err_topic = r.flags.as<unsigned>();
        const int rc = launch_stage_plan<false>(c, s, p, pl, d.T, 0, 1 << c->br.lut_mode);
        if (rc != KA_OK) return rc;
    }
    const bool tables = pl.a_levels && d.T > 0;
    if (done && !tables) KA_CUDA(cudaEventRecord(done, s));
    if (c->timing) KA_CUDA(cudaEventRecord(a_done, s));
    if (tables) {
        int32_t* ntl = r.ntl.as<int32_t>() + d.topic_base;
        int32_t* loff = r.loff.as<int32_t>() + d.topic_base + d.blk;  // every block keeps T_k + 1 entries
        ka_level_scan_kernel<<<1, 1024, 0, s>>>(ntl, d.T, loff);
        KA_CUDA(cudaGetLastError());
        ka_level_fill_kernel<<<(d.T + 7) / 8, 256, 0, s>>>(ntl, loff, r.lend.as<uint32_t>() + d.q0, d.d_part_off, d.P, d.T, d.T, d.Q,
                                                            r.lvl_end.as<uint32_t>() + d.q0);
        KA_CUDA(cudaGetLastError());
        c->launches += 2;
        if (done) KA_CUDA(cudaEventRecord(done, s));
    }
    return KA_OK;
}

// CAND: one CTA per candidate of a batched solve (ncand of them), else one CTA. behind: launched behind the kernel before it
// on s (programmatic dependent launch): the chain's prologue overlaps that kernel's end, and only its counter load waits for
// it. Only for a predecessor that writes none of the records the chain reads.
template <int KIND, int MAXNT, bool CAND, bool GCTR, bool SINGLE, bool WARP1, bool FULL>
cudaError_t launch_order_t(cudaStream_t s, const KaOrderParams& o, const Plan& pl, int ncand, bool behind) {
    auto kern = ka_order_levels_kernel<KIND, GCTR, MAXNT, SINGLE, WARP1, FULL, CAND>;
    cudaError_t e = allow_smem(kern, pl.b_smem);
    if (e != cudaSuccess) return e;
    cudaLaunchAttribute attr{};
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(CAND ? ncand : 1);
    cfg.blockDim = dim3(pl.b_threads);
    cfg.dynamicSmemBytes = pl.b_smem;
    cfg.stream = s;
    cfg.attrs = &attr;
    cfg.numAttrs = behind ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, o);
}

// KIND 0 / 1: slot chains of rows <= 3 (chunk arithmetic, barrier flavour, full chunks are compile-time); 4 / 8: rows of 4 / 5..8.
// *sel: the instantiation launched, (GCTR ? 4 : 0) | loop shape (0 general, 1 WARP1, 2 SINGLE, 3 FULL).
template <int KIND, int MAXNT, bool CAND = false>
cudaError_t launch_order(cudaStream_t s, const KaOrderParams& o, const Plan& pl, int* sel, int ncand = 0, bool behind = false) {
    if constexpr (KIND > 1) {
        *sel = pl.b_gctr ? 4 : 0;
        return pl.b_gctr ? launch_order_t<KIND, MAXNT, false, true, false, false, false>(s, o, pl, ncand, behind)
                         : launch_order_t<KIND, MAXNT, false, false, false, false, false>(s, o, pl, ncand, behind);
    } else {
        const bool warp1 = pl.b_threads == 32;                                                          // window mode
        const bool single = !warp1 && o.uniform_width != 0 && o.uniform_width <= (uint32_t)pl.b_threads;   // chunk = topic
        const bool full = single && o.uniform_width == (uint32_t)pl.b_threads;                          // no idle lane
        *sel = (pl.b_gctr ? 4 : 0) | (warp1 ? 1 : (full ? 3 : (single ? 2 : 0)));
        switch (*sel) {
            case 0: return launch_order_t<KIND, MAXNT, CAND, false, false, false, false>(s, o, pl, ncand, behind);
            case 1: return launch_order_t<KIND, MAXNT, CAND, false, false, true, false>(s, o, pl, ncand, behind);
            case 2: return launch_order_t<KIND, MAXNT, CAND, false, true, false, false>(s, o, pl, ncand, behind);
            case 3: return launch_order_t<KIND, MAXNT, CAND, false, true, false, true>(s, o, pl, ncand, behind);
            case 4: return launch_order_t<KIND, MAXNT, CAND, true, false, false, false>(s, o, pl, ncand, behind);
            case 5: return launch_order_t<KIND, MAXNT, CAND, true, false, true, false>(s, o, pl, ncand, behind);
            case 6: return launch_order_t<KIND, MAXNT, CAND, true, true, false, false>(s, o, pl, ncand, behind);
            default: return launch_order_t<KIND, MAXNT, CAND, true, true, false, true>(s, o, pl, ncand, behind);
        }
    }
}

// ka_ctx_last_order_plan: a chain launch of the current solve call (sel as launch_order reports it, ncand 0 for a single solve).
void note_order(ka_ctx* c, const Plan& pl, int sel, int ncand) {
    int32_t* r = c->order_plan;
    r[0] = pl.rec_kind;
    r[1] = pl.a_levels;
    r[2] = pl.b_threads;
    r[3] = pl.b_ring_log2;
    r[4] = (sel >> 2) & 1;
    r[5] = sel & 3;
    r[6]++;
    r[7] = ncand;
}

// Topics per chain sub-block of a large block (at least KA_CHAIN_LARGE_BLOCK topics) of a single solve, whose chain launches
// overlap (enq_order_emit). A solve ends about one sub-block's slot-1 chain after its slot-0 chain ends, so smaller sub-blocks
// shorten that tail; but a slot-1 chain launch waits for its slot-0 chain (an event), which keeps it from overlapping the
// slot-1 chain before it: measured at C3 on H100, a slot-1 boundary costs about 7 us against 3 us for a slot-0 one, while a
// slot-1 level is about 7 ns faster. Below about 650 levels per sub-block the slot-1 chain falls further behind at every
// boundary (DESIGN §2 "Pipelining").
constexpr int KA_CHAIN_SUB_TOPICS = 512;
constexpr int KA_CHAIN_LARGE_BLOCK = 1024;

// How many topic sub-blocks the slot chains of one staged block are cut into: the slot-0 chain of sub-block j+1 runs (on
// its own SM) while the slot-1 chain + emit of sub-block j run. A chain launch is one CTA, so sub-blocks are cheap; each
// should still hold a few hundred levels to amortise the launch + ring fill. overlapped: the chain launches of the
// sub-blocks overlap their predecessors (the single solve), which makes a boundary cheap enough for many sub-blocks.
int chain_subblocks(const StageDesc& d, int blocks_in_solve, bool overlapped = false) {
    if (d.d_part_off || d.pl.rec_kind != 3 || d.T < 2) return 1;
    int n = std::max(1, 8 / std::max(1, blocks_in_solve));
    n = std::min(n, std::max(1, d.T / 128));
    if (overlapped && d.T >= KA_CHAIN_LARGE_BLOCK) n = std::max(n, d.T / KA_CHAIN_SUB_TOPICS);
    if (const char* e = std::getenv("KA_CHAIN_SUBBLOCKS")) n = std::max(1, std::min(std::atoi(e), d.T));
    return std::min(n, KA_MAX_CHAIN_BLOCKS);
}

// Per-call state of one solve: where its inputs come from and its rows go, and how far its enqueue has got. Lives on the
// stack of the entry point.
struct SolveCall {
    // host-buffer entry points: inputs of the whole problem in host memory, copied H2D block by block (null: on the device)
    const int32_t* h_hash = nullptr;
    const int32_t* h_cur = nullptr;
    const int64_t* h_part_off = nullptr;  // ragged
    const int64_t* h_rep_off = nullptr;
    const int32_t* h_part_id = nullptr;   // ragged JSON solve: partition ids, copied to d_part_id (the text prints them)
    int32_t* d_part_id = nullptr;
    // rows of the whole problem on the device, and their host destination (null: they stay on the device)
    int32_t* d_out = nullptr;
    int32_t* d_out_len = nullptr;
    int32_t* h_out = nullptr;
    int32_t* h_out_len = nullptr;
    bool json = false;        // ka_solve_dense_json / ka_solve_json: rows -> JSON text on c->sj as soon as they are final
    // pipelined host-buffer solve, rows <= 3: every chain sub-block is copied out on c->sj as soon as its emit is done, so
    // that no D2H sits between two slot-1 chains on the caller's stream
    bool stream_out = false;
    int json_blocks = 0;      // JSON fragments enqueued (ev_json_in, ev_json_scan, h_frag)
    int chains = 0;           // chain sub-blocks enqueued (ev_b1, ev_b2)
    bool emits = false;       // emits enqueued on c->sj (ev_emit_done)

    SolveCall(int32_t* out, int32_t* out_len) : d_out(out), d_out_len(out_len) {}
};

// A host-buffer solve: its inputs from these host arrays (part_id: a ragged JSON solve's partition ids), its rows to the ctx's
// d_out / d_out_len and then to out_broker / out_len (null: no host rows). Made once the ctx's device buffers are reserved.
SolveCall host_call(ka_ctx* c, const int32_t* topic_hash, const int64_t* part_off, const int64_t* rep_off, const int32_t* cur_broker,
                    int32_t* out_len, int32_t* out_broker, const int32_t* part_id = nullptr) {
    SolveCall io(c->d_out.as<int32_t>(), c->d_out_len.as<int32_t>());
    io.h_hash = topic_hash;
    io.h_part_off = part_off;
    io.h_rep_off = rep_off;
    io.h_cur = cur_broker;
    io.h_part_id = part_id;
    io.d_part_id = part_id ? c->d_part_id.as<int32_t>() : nullptr;
    io.h_out = out_broker;
    io.h_out_len = out_len;
    return io;
}

struct SubBlock { int t0, t1; int64_t r0, rq; };

SubBlock sub_block(const StageDesc& d, int j, int nsub) {
    SubBlock b;
    b.t0 = (int)((int64_t)d.T * j / nsub);
    b.t1 = (int)((int64_t)d.T * (j + 1) / nsub);
    // ragged blocks are never cut (nsub == 1): sub-block rows follow from the dense shape
    b.r0 = d.d_part_off ? 0 : (int64_t)b.t0 * d.P;
    b.rq = d.d_part_off ? d.Q : (int64_t)(b.t1 - b.t0) * d.P;
    return b;
}

// A text pass over rows [row0, row0 + rows) of out / out_len (stride S), laid out as T topics (ragged: part_off and, when
// given, part_id), printed with the ctx's name slab into its text buffer, cap bytes of it.
KaJsonParams json_params(ka_ctx* c, const int32_t* out, const int32_t* out_len, int S, int T, const int64_t* part_off,
                         const int32_t* part_id, int64_t row0, int64_t rows, unsigned long long cap) {
    KaJsonParams p{};
    p.Q = (uint32_t)rows;
    p.row0 = (uint32_t)row0;
    p.T = T;
    p.part_off = part_off;
    p.part_id = part_id;
    p.name_off = c->d_name_off.as<int64_t>();
    p.names = c->d_names.as<char>();
    p.out = out + row0 * S;
    p.out_len = out_len + row0;
    p.S = S;
    p.rowlen = c->d_json_rowlen.as<uint32_t>() + row0;
    p.json = c->d_json.as<char>();
    p.cap = cap;
    return p;
}

// Fragment k of a solve's text (block d, rows in io): rows [row0, row0 + rows), their block sums, and slot k of the running
// text state.
KaJsonParams json_fragment(ka_ctx* c, const StageDesc& d, const SolveCall& io, int64_t row0, int64_t rows, int k) {
    KaJsonParams p = json_params(c, io.d_out, io.d_out_len, d.S, d.T, d.d_part_off, io.d_part_id, row0, rows,
                                 (unsigned long long)c->d_json.cap);
    p.blocksum = c->d_json_blocksum.as<uint32_t>() + (row0 / 256) + k;
    p.total = c->d_json_state.as<unsigned long long>();
    p.frag = p.total + 2 + 2 * k;
    return p;
}

// The length pass and the scan of fragment p on s (SEG: of a fleet, with its document table sg).
template <bool SEG>
void enq_json_lengths(cudaStream_t s, const KaJsonParams& p, const KaJsonSegs& sg) {
    const int nblocks = (int)((p.Q + 255) / 256);
    if (nblocks > 0) ka_json_len_kernel<SEG><<<nblocks, 256, 0, s>>>(p, sg);
    ka_json_scan_kernel<<<1, 1024, 0, s>>>(p, nblocks);
}

// A write pass of the text passes: `grid` CTAs of 256 threads with the shared-memory stage, on s.
template <typename K, typename... A>
cudaError_t enq_json_write(K kernel, unsigned grid, cudaStream_t s, const A&... args) {
    const cudaError_t e = allow_smem(kernel, KA_JSON_SMEM_BYTES + 16);
    if (e == cudaSuccess) kernel<<<grid, 256, KA_JSON_SMEM_BYTES + 16, s>>>(args...);
    return e;
}

// KAG:169-186 for a finished range of rows (sub-block b of block d): rows -> JSON text at the running offset of d_json, on c->sj.
int enq_json_rows(ka_ctx* c, cudaStream_t s_done, SolveCall& io, const StageDesc& d, const SubBlock& b, bool first, bool last) {
    const int k = io.json_blocks;
    if (k >= KA_MAX_JSON_FRAGS) return KA_ERR_LIMIT;
    KA_CUDA(cudaEventRecord(c->ev_json_in[k], s_done));
    KA_CUDA(cudaStreamWaitEvent(c->sj, c->ev_json_in[k], 0));
    KaJsonParams p = json_fragment(c, d, io, d.q0 + b.r0, b.rq, k);
    p.P = std::max(d.P, 1);
    p.topic0 = d.topic_base + b.t0;
    p.first = first;
    p.last = last;
    enq_json_lengths<false>(c->sj, p, KaJsonSegs{});
    KA_CUDA(enq_json_write(ka_json_write_kernel<false>, std::max((p.Q + 255) / 256, 1u), c->sj, p, KaJsonSegs{}));
    KA_CUDA(cudaGetLastError());
    KA_CUDA(cudaMemcpyAsync(c->h_frag + 2 * k, p.frag, 16, cudaMemcpyDeviceToHost, c->sj));
    KA_CUDA(cudaEventRecord(c->ev_json_scan[k], c->sj));
    c->launches += 3;
    io.json_blocks = k + 1;
    return KA_OK;
}

// Rows per JSON fragment of a ragged solve of Q rows (a multiple of 256: fragments own whole blocks of the length pass).
int64_t json_fragment_rows(int64_t Q) {
    const int64_t spread = (Q + KA_MAX_JSON_FRAGS - 1) / KA_MAX_JSON_FRAGS;
    return std::max(KA_JSON_FRAG_ROWS, (spread + 255) / 256 * 256);
}

// JSON of the finished rows of sub-block b. A ragged block is never cut into chain sub-blocks, so its text is cut into
// fragments here instead; a ragged run without rows still gets its (empty) text.
int enq_json(ka_ctx* c, cudaStream_t s_done, SolveCall& io, const StageDesc& d, const SubBlock& b, bool first, bool last) {
    if (!d.d_part_off) return enq_json_rows(c, s_done, io, d, b, first, last);
    const int64_t step = json_fragment_rows(b.rq);
    int64_t r = 0;
    do {
        SubBlock f = b;
        f.r0 = b.r0 + r;
        f.rq = std::min(step, b.rq - r);
        const int rc = enq_json_rows(c, s_done, io, d, f, first && r == 0, last && r + step >= b.rq);
        if (rc != KA_OK) return rc;
        r += step;
    } while (r < b.rq);
    return KA_OK;
}

// D2H of rows [r0, r0 + rows) of a solve's output.
int enq_copy_out(cudaStream_t s, const SolveCall& io, int S, int64_t r0, int64_t rows) {
    KA_CUDA(cudaMemcpyAsync(io.h_out + r0 * S, io.d_out + r0 * S, (size_t)rows * S * 4, cudaMemcpyDeviceToHost, s));
    if (io.h_out_len) KA_CUDA(cudaMemcpyAsync(io.h_out_len + r0, io.d_out_len + r0, (size_t)rows * 4, cudaMemcpyDeviceToHost, s));
    return KA_OK;
}

// Leader-order parameters of sub-block b of a staged block.
KaOrderParams order_params(ka_ctx* c, const StageDesc& d, const SubBlock& b) {
    const Plan& pl = d.pl;
    KaOrderParams o{};
    o.N = c->br.N;
    o.S = d.S;
    o.uniform_width = pl.a_levels ? 0u : (uint32_t)d.P;
    o.chunk_end = pl.a_levels ? c->run.lvl_end.as<uint32_t>() + d.q0 : nullptr;
    o.ctr8 = c->d_ctr8.as<int32_t>();
    o.ring_log2 = pl.b_ring_log2;
    const int32_t* loff = pl.a_levels ? c->run.loff.as<int32_t>() + d.topic_base + d.blk : nullptr;
    o.Q = (uint32_t)b.rq;
    o.rec = c->run.rec.as<unsigned char>() + (size_t)(d.q0 + b.r0) * pl.rec_bytes;
    o.pos_base = (uint32_t)b.r0;
    o.chunk_lo_ptr = loff ? loff + b.t0 : nullptr;
    o.chunk_hi_ptr = loff ? loff + b.t1 : nullptr;
    return o;
}

// One slot chain (rows <= 3) over sub-block j of a staged block; behind: as launch_order_t.
int enq_slot_chain(ka_ctx* c, cudaStream_t s, const StageDesc& d, int slot, int j, int nsub, bool behind = false) {
    const SubBlock b = sub_block(d, j, nsub);
    if (b.rq <= 0 || c->br.N <= 0) return KA_OK;
    const KaOrderParams o = order_params(c, d, b);
    int sel = 0;
    KA_CUDA((slot == 0 ? launch_order<0, 1024>(s, o, d.pl, &sel, 0, behind) : launch_order<1, 1024>(s, o, d.pl, &sel, 0, behind)));
    note_order(c, d.pl, sel, 0);
    c->launches++;
    return KA_OK;
}

// Emit of sub-block j (rows <= 3): ordered records -> broker ids, list lengths, slot-2 counters.
int enq_emit_block(ka_ctx* c, cudaStream_t s, const StageDesc& d, int j, int nsub, int32_t* d_out, int32_t* d_out_len) {
    const Plan& pl = d.pl;
    const SubBlock b = sub_block(d, j, nsub);
    if (b.rq <= 0 || c->br.N <= 0) return KA_OK;
    ka_emit3_kernel<<<(unsigned)((b.rq + 255) / 256), 256, 0, s>>>(
        reinterpret_cast<const uint4*>(c->run.rec.as<unsigned char>() + (size_t)(d.q0 + b.r0) * pl.rec_bytes),
        pl.a_levels ? c->run.perm.as<uint16_t>() + d.q0 + b.r0 : nullptr, d.d_part_off, b.t1 - b.t0, d.P, c->d_broker_id.as<int32_t>(),
        (uint32_t)b.rq, d.S, d_out + (size_t)b.r0 * d.S, d_out_len ? d_out_len + b.r0 : nullptr, c->d_ctr8.as<int32_t>());
    KA_CUDA(cudaGetLastError());
    c->launches++;
    return KA_OK;
}

// The serial chains through Context.counter (KAS:202-239) for a staged block + the parallel emit into the block's rows of
// io.d_out. Rows <= 3: slot-0 chains on c->sb1, slot-1 chains on `s`, emits (and the rows' copy-out or text) on c->sj; the
// caller has made c->sb1 wait for the stage (c->ev_chain_in recorded after kernel A / the counter import), and joins the
// emits back into `s` (join_emits) once every block is enqueued. next_stage (a pipelined solve's next block: its kernel A
// is done): c->sb1 waits for it before this block's last slot-0 chain rather than before the next block's first one, so
// that one is launched behind its stream predecessor like the chains inside a block. That kernel A ends long before.
int enq_order_emit(ka_ctx* c, cudaStream_t s, const StageDesc& d, SolveCall& io, int blocks_in_solve, cudaEvent_t next_stage = nullptr) {
    const int S = d.S;
    const Plan& pl = d.pl;
    if (next_stage && (d.Q <= 0 || c->br.N <= 0 || pl.rec_kind != 3)) KA_CUDA(cudaStreamWaitEvent(c->sb1, next_stage, 0));
    if (d.Q <= 0 || c->br.N <= 0) return io.json && d.d_part_off && d.Q == 0 ? enq_json(c, s, io, d, sub_block(d, 0, 1), true, true) : KA_OK;
    int32_t* d_out = io.d_out + d.q0 * S;
    int32_t* d_out_len = io.d_out_len ? io.d_out_len + d.q0 : nullptr;
    if (pl.rec_kind != 3) {  // rows of 4..8: one fused chain over all slots, rows written by the kernel
        const SubBlock b = sub_block(d, 0, 1);
        KaOrderParams o = order_params(c, d, b);
        o.broker_id = c->d_broker_id.as<int32_t>();
        o.out = d_out;
        o.out_len = d_out_len;
        int sel = 0;
        KA_CUDA((pl.rec_kind == 4 ? launch_order<4, 512>(s, o, pl, &sel) : launch_order<8, 256>(s, o, pl, &sel)));
        note_order(c, pl, sel, 0);
        c->launches++;
        if (io.json) return enq_json(c, s, io, d, b, d.blk == 0, d.blk == blocks_in_solve - 1);
        return KA_OK;
    }
    const int nsub = chain_subblocks(d, blocks_in_solve, true);
    const int e = c->chain_used;
    if (e >= KA_MAX_BLOCKS || io.chains + nsub > KA_MAX_CHAIN_EVENTS) return KA_ERR_LIMIT;
    // Each chain stream runs the chains of the block back to back, every one launched behind the one before it: its prologue
    // overlaps that chain's end. The slot-1 chains read records the slot-0 chains rewrote, and the emits read the slot-1
    // chains' records, so each hands over through an event (ev_b1, ev_b2); the emits run on c->sj, off the slot-1 path.
    cudaStream_t s1 = c->sb1, se = c->sj;
    const int jw = nsub > 1 ? nsub - 1 : nsub;   // next_stage is waited for before slot-0 chain jw (nsub: after the block)
    // The slot-0 chains are timed from the first block's start to the last block's end (ev_chain[0][0..1]): a timed event
    // record between two blocks' chains would keep the second from launching behind the first.
    if (c->timing && e == 0) KA_CUDA(cudaEventRecord(c->ev_chain[0][0], s1));
    for (int j = 0; j < nsub; ++j) {
        const int k = io.chains + j;
        if (next_stage && j == jw) KA_CUDA(cudaStreamWaitEvent(s1, next_stage, 0));
        int rc = enq_slot_chain(c, s1, d, 0, j, nsub, true);              // slot-0 chain
        if (rc != KA_OK) return rc;
        KA_CUDA(cudaEventRecord(c->ev_b1[k], s1));
        KA_CUDA(cudaStreamWaitEvent(s, c->ev_b1[k], 0));
        if (c->timing && j == 0 && e == 0) KA_CUDA(cudaEventRecord(c->ev_chain[0][2], s));   // as slot 0: one span per solve
        if ((rc = enq_slot_chain(c, s, d, 1, j, nsub, true)) != KA_OK) return rc;   // slot-1 chain
        KA_CUDA(cudaEventRecord(c->ev_b2[k], s));
        KA_CUDA(cudaStreamWaitEvent(se, c->ev_b2[k], 0));
        if ((rc = enq_emit_block(c, se, d, j, nsub, d_out, d_out_len)) != KA_OK) return rc;
        if (j == nsub - 1) {   // the block's emits are done: join_emits hands them to `s`
            if (c->timing) KA_CUDA(cudaEventRecord(c->ev_chain[0][3], se));   // the last block's record ends the span
            KA_CUDA(cudaEventRecord(c->ev_emit_done, se));
            io.emits = true;
        }
        const SubBlock b = sub_block(d, j, nsub);
        // the rows of this sub-block are final: copy them out, or build and stream out their JSON text
        if (io.stream_out && (rc = enq_copy_out(se, io, S, d.q0 + b.r0, b.rq)) != KA_OK) return rc;
        if (io.json && (rc = enq_json(c, se, io, d, b, d.blk == 0 && j == 0, d.blk == blocks_in_solve - 1 && j == nsub - 1)) != KA_OK)
            return rc;
    }
    if (next_stage && jw == nsub) KA_CUDA(cudaStreamWaitEvent(s1, next_stage, 0));
    if (c->timing && !next_stage) KA_CUDA(cudaEventRecord(c->ev_chain[0][1], s1));
    io.chains += nsub;
    c->chain_used = e + 1;
    return KA_OK;
}

// `s` waits for every emit enq_order_emit put on c->sj (not for the copies and text behind them).
int join_emits(ka_ctx* c, cudaStream_t s, const SolveCall& io) {
    if (io.emits) KA_CUDA(cudaStreamWaitEvent(s, c->ev_emit_done, 0));
    return KA_OK;
}

// c->sb1 (slot-0 chain stream) must see everything enqueued on `s` so far: the staged records / imported counters
int chain_fork(ka_ctx* c, cudaStream_t s) {
    KA_CUDA(cudaEventRecord(c->ev_chain_in, s));
    KA_CUDA(cudaStreamWaitEvent(c->sb1, c->ev_chain_in, 0));
    return KA_OK;
}

// End of a solve on `s`: status words back to pinned host memory (async), end of the timed span.
int enq_solve_end(ka_ctx* c, cudaStream_t s) {
    KA_CUDA(cudaMemcpyAsync(&c->h_pin->err_topic, c->run.flags.p, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (c->timing) {
        KA_CUDA(cudaEventRecord(c->ev[5], s));
        c->ev_valid = true;
    }
    return KA_OK;
}

// How many topic super-chunks a dense solve is pipelined in (1 = no pipelining).
int pipeline_stages(int T, int64_t Q) {
    // worthwhile only when every chunk still has enough topics to keep kernel A throughput-bound (a topic is one warp:
    // with few topics per chunk A is latency-bound and K chunks cost K times as much — measured on config 5)
    int k = Q >= 262144 ? std::min(4, T / 2048) : 1;
    if (const char* e = std::getenv("KA_PIPELINE_STAGES")) k = std::atoi(e);
    return std::max(1, std::min(k, std::min(KA_MAX_BLOCKS, std::max(T, 1))));
}

// H2D of the host inputs of block d (ncur current replicas).
int enq_inputs(cudaStream_t s, const SolveCall& io, const StageDesc& d, int64_t ncur) {
    // the destinations are the ctx's scratch copies (a host-buffer solve's StageDesc points into them)
    auto h2d = [&](const void* dst, const void* src, size_t bytes) {
        return cudaMemcpyAsync(const_cast<void*>(dst), src, bytes, cudaMemcpyHostToDevice, s);
    };
    if (io.h_hash && d.T > 0) KA_CUDA(h2d(d.d_hash, io.h_hash + d.topic_base, (size_t)d.T * 4));
    if (io.h_part_off && d.T > 0) KA_CUDA(h2d(d.d_part_off, io.h_part_off, (size_t)(d.T + 1) * 8));
    if (io.h_rep_off && d.Q > 0) KA_CUDA(h2d(d.d_rep_off, io.h_rep_off, (size_t)(d.Q + 1) * 8));
    if (io.h_part_id && d.Q > 0) KA_CUDA(h2d(io.d_part_id, io.h_part_id, (size_t)d.Q * 4));
    if (io.h_cur && ncur > 0) KA_CUDA(h2d(d.d_cur, io.h_cur + d.q0 * d.RF, (size_t)ncur * 4));
    return KA_OK;
}

// A whole solve on the caller's stream `s`: H2D -> flags reset -> stage -> chain fork -> order/emit -> copy-out -> flags
// readback. Dense problems large enough are pipelined in K topic super-chunks: c->aux runs (the H2D,) kernel A and the
// level tables of chunk k+1 while `s` runs the leader-order chains of chunk k (and the D2H of its output); `s` orders the
// chunks strictly one after the other through the counters in ctr8.
int run_solve(ka_ctx* c, cudaStream_t s, const Shape& sh, SolveCall& io, ka_status* st) {
    c->staged = false;   // the solve reuses the scratch a staged block lives in
    c->last_was_staged = false;
    reset_plans(c);
    const bool ragged = sh.d_part_off != nullptr;
    const int T = sh.T;
    const int K = ragged ? 1 : pipeline_stages(T, (int64_t)T * sh.P);
    // Block boundaries: the first block's H2D and the last block's D2H are the only copies that nothing overlaps, so with
    // host buffers the end blocks get half the weight of the inner ones (1:2:..:2:1).
    const bool host_io = (io.h_cur != nullptr || io.h_out != nullptr) && K >= 3;
    const int wsum = host_io ? 2 * (K - 1) : K;
    auto bound = [&](int k) { return k <= 0 ? 0 : (k >= K ? T : (int)((int64_t)T * (host_io ? 2 * k - 1 : k) / wsum)); };
    StageDesc ds[KA_MAX_BLOCKS];
    int rc;
    for (int k = 0; k < K; ++k)
        if ((rc = describe_block(sh, bound(k), bound(k + 1), k, c->br.N, c->br.blob_bytes, ds[k], st)) != KA_OK) return rc;
    if ((rc = reserve_scratch(c, ds, K)) != KA_OK) return rc;
    c->last_stages = K;
    if (c->timing) KA_CUDA(cudaEventRecord(c->ev[0], s));
    if (K == 1) {
        const StageDesc& d = ds[0];
        if ((rc = enq_inputs(s, io, d, ragged ? sh.R : d.Q * d.RF)) != KA_OK) return rc;
        if ((rc = reset_flags(c, s)) != KA_OK) return rc;
        if (c->timing) KA_CUDA(cudaEventRecord(c->ev[1], s));
        if ((rc = enq_stage(c, s, d, c->ev[2])) != KA_OK) return rc;
        if (c->timing) KA_CUDA(cudaEventRecord(c->ev[3], s));
        if ((rc = chain_fork(c, s)) != KA_OK) return rc;
        if ((rc = enq_order_emit(c, s, d, io, 1)) != KA_OK || (rc = join_emits(c, s, io)) != KA_OK) return rc;
        if (c->timing) KA_CUDA(cudaEventRecord(c->ev[4], s));
        if (io.h_out && d.Q > 0 && c->br.N > 0 && (rc = enq_copy_out(s, io, d.S, 0, d.Q)) != KA_OK) return rc;
    } else {
        cudaStream_t aux = c->aux;
        io.stream_out = io.h_out && ds[0].pl.rec_kind == 3 && !io.json;
        KA_CUDA(cudaEventRecord(c->ev_in, s));           // inputs ready / earlier work on s done
        if (io.stream_out) KA_CUDA(cudaStreamWaitEvent(c->sj, c->ev_in, 0));
        KA_CUDA(cudaStreamWaitEvent(aux, c->ev_in, 0));
        if ((rc = reset_flags(c, aux)) != KA_OK) return rc;
        // every block's stage is enqueued before the chains: enqueueing a block's chains takes the host longer than kernel A
        // of the next block takes the GPU, so a stage enqueued behind them would start late and hold up the next block's chains
        for (int k = 0; k < K; ++k) {
            const StageDesc& d = ds[k];
            if ((rc = enq_inputs(aux, io, d, d.Q * d.RF)) != KA_OK) return rc;
            if (c->timing) KA_CUDA(cudaEventRecord(c->ev_pipe[k][0], aux));
            if ((rc = enq_stage(c, aux, d, c->ev_pipe[k][1], c->ev_stage[k])) != KA_OK) return rc;
            if (c->timing) KA_CUDA(cudaEventRecord(c->ev_pipe[k][2], aux));
        }
        for (int k = 0; k < K; ++k) {
            const StageDesc& d = ds[k];
            KA_CUDA(cudaStreamWaitEvent(s, c->ev_stage[k], 0));
            if (k == 0) {   // c->sb1 waits for the later blocks' stages inside enq_order_emit
                KA_CUDA(cudaStreamWaitEvent(c->sb1, c->ev_stage[0], 0));
                KA_CUDA(cudaStreamWaitEvent(c->sb1, c->ev_in, 0));
            }
            // chains of all blocks timed as one span: a timed record between two blocks' slot-1 chains delays the second
            if (c->timing && k == 0) KA_CUDA(cudaEventRecord(c->ev_pipe[0][3], s));
            if ((rc = enq_order_emit(c, s, d, io, K, k + 1 < K ? c->ev_stage[k + 1] : nullptr)) != KA_OK) return rc;
            if (c->timing && k == K - 1) KA_CUDA(cudaEventRecord(c->ev_pipe[K - 1][4], s));
            // rows of 4..8: one copy per block on the caller's stream
            if (io.h_out && !io.stream_out && d.Q > 0 && c->br.N > 0 && (rc = enq_copy_out(s, io, d.S, d.q0, d.Q)) != KA_OK) return rc;
        }
        if ((rc = join_emits(c, s, io)) != KA_OK) return rc;
        if (io.stream_out) {   // join the copy-out stream back into the caller's stream
            KA_CUDA(cudaEventRecord(c->ev_out_done, c->sj));
            KA_CUDA(cudaStreamWaitEvent(s, c->ev_out_done, 0));
        }
    }
    return enq_solve_end(c, s);
}

// The status a run reports for its lowest failing topic t, whose tstatus entry is ts. part_id / part_off (ragged
// host-buffer solve): the reported partition is the failing partition's id rather than its ordinal inside the topic.
ka_status topic_status(int t, const int4& ts, const int32_t* part_id, const int64_t* part_off) {
    ka_status r;
    set_status(&r, ts.x, t, ts.y >= 0 && part_id && part_off ? part_id[part_off[t] + ts.y] : ts.y, ts.z, ts.w);
    return r;
}

// Wait for the stream, translate device flags into a ka_status. part_id / part_off: as in topic_status.
int finish_status(ka_ctx* c, cudaStream_t s, ka_status* st, const int32_t* part_id = nullptr, const int64_t* part_off = nullptr) {
    KA_CUDA(cudaStreamSynchronize(s));
    c->pending_status = false;
    ka_status r{};
    set_status(&r, KA_OK);
    if (c->h_pin->err_topic != -1) {
        const int t = c->h_pin->err_topic;
        KA_CUDA(cudaMemcpy(&c->h_pin->tstatus, c->run.tstatus.as<int4>() + t, sizeof(int4), cudaMemcpyDeviceToHost));
        r = topic_status(t, c->h_pin->tstatus, part_id, part_off);
        r.topic_index += c->last_was_staged ? c->topic_base : 0;
    }
    if (c->timing && c->ev_valid) {
        for (int i = 0; i < 8; ++i) c->last_ms[i] = 0.f;
        cudaEventElapsedTime(&c->last_ms[5], c->ev[0], c->ev[5]);  // total on the stream
        if (c->last_stages <= 1) {
            cudaEventElapsedTime(&c->last_ms[3], c->ev[0], c->ev[1]);  // H2D
            cudaEventElapsedTime(&c->last_ms[0], c->ev[1], c->ev[2]);  // kernel A
            cudaEventElapsedTime(&c->last_ms[1], c->ev[2], c->ev[3]);  // level tables (scan + fill; absent when capacity is 1)
            cudaEventElapsedTime(&c->last_ms[7], c->ev[3], c->ev[4]);  // all chains + emit, wall time on the stream
            cudaEventElapsedTime(&c->last_ms[4], c->ev[4], c->ev[5]);  // D2H
        } else {  // pipelined: phases of different chunks overlap; report the per-phase sums
            for (int k = 0; k < c->last_stages; ++k) {
                float a = 0.f, t = 0.f;
                cudaEventElapsedTime(&a, c->ev_pipe[k][0], c->ev_pipe[k][1]);
                cudaEventElapsedTime(&t, c->ev_pipe[k][1], c->ev_pipe[k][2]);
                c->last_ms[0] += a;
                c->last_ms[1] += t;
            }
            cudaEventElapsedTime(&c->last_ms[7], c->ev_pipe[0][3], c->ev_pipe[c->last_stages - 1][4]);
        }
        if (c->chain_used > 0) {  // rows <= 3: each slot's chains, first start .. last end (slot 1 with its emits)
            cudaEventElapsedTime(&c->last_ms[2], c->ev_chain[0][0], c->ev_chain[0][1]);
            cudaEventElapsedTime(&c->last_ms[6], c->ev_chain[0][2], c->ev_chain[0][3]);
        } else if (c->slot_timed[0] || c->slot_timed[1]) {  // per-slot entry points (topic-sharded runs)
            if (c->slot_timed[0]) cudaEventElapsedTime(&c->last_ms[2], c->ev_chain[0][0], c->ev_chain[0][1]);
            if (c->slot_timed[1]) cudaEventElapsedTime(&c->last_ms[6], c->ev_chain[1][0], c->ev_chain[1][1]);
        } else {
            c->last_ms[2] = c->last_ms[7];  // rows of 4..8: one fused chain
        }
    }
    c->last = r;
    if (st) *st = r;
    return r.code;
}

// Prologue of an entry point: the ctx's device current and, with `collect`, the status of the previous asynchronous solve
// collected first (it may have run on another stream than this call's).
int enter(ka_ctx* c, bool collect) {
    KA_CUDA(cudaSetDevice(c->device));
    if (collect && c->pending_status) finish_status(c, c->last_stream, nullptr);
    return KA_OK;
}

// Wait for the last asynchronous call that left no status pending (end_untracked).
int wait_untracked(ka_ctx* c) {
    if (!c->tail_pending) return KA_OK;
    KA_CUDA(cudaEventSynchronize(c->ev_tail));
    c->tail_pending = false;
    return KA_OK;
}

// Prologue of a host call, whose work runs on the ctx's own streams, the legacy stream or the host, none of which is ordered
// after the caller's stream: enter(c, true), then wait_untracked. So the host call sees every earlier call of the ctx, and
// nothing it writes reaches what such a call still has to read.
int enter_host(ka_ctx* c) {
    const int rc = enter(c, true);
    return rc != KA_OK ? rc : wait_untracked(c);
}

// End of an asynchronous call that leaves no status pending, its work enqueued on `s`: recorded there for the next host call
// to wait for. The call itself does not wait.
int end_untracked(ka_ctx* c, cudaStream_t s) {
    KA_CUDA(cudaEventRecord(c->ev_tail, s));
    c->tail_pending = true;
    return KA_OK;
}

// Everything of a solve is enqueued on `s`: its status is pending until ka_last_status, or collected now when the caller
// asked for it (st) or the entry point is synchronous.
int finish(ka_ctx* c, cudaStream_t s, ka_status* st, bool sync, const int32_t* part_id = nullptr, const int64_t* part_off = nullptr) {
    c->last_stream = s;
    c->pending_status = true;
    return st || sync ? finish_status(c, s, st, part_id, part_off) : KA_OK;
}

// A library-side failure of a batched solve: every member reports it.
int fail_members(ka_status* st, int K, int rc) {
    for (int k = 0; k < K; ++k) set_status(st + k, rc);
    return rc;
}

// A batched solve failed with rc after part of it was enqueued on `s` (slot-0 chains on c->sb1): wait for what was enqueued,
// then every member reports rc.
int abort_batch(ka_ctx* c, cudaStream_t s, ka_status* st, int K, int rc) {
    cudaStreamSynchronize(c->sb1);
    cudaStreamSynchronize(s);
    return fail_members(st, K, rc);
}

// The checks every batched call starts with. Without st or with K < 0 there is nowhere to report; otherwise every st[k] starts
// at KA_OK and the first of these failures fails every member: no ctx, K beyond the limit or rows wider than 3 (the batched
// chains are the slot chains of rows <= 3; wider rows take the single solve's fused chain), out_stride < 1.
int batch_args(ka_ctx* c, int K, int out_stride, ka_status* st) {
    if (!st || K < 0) return KA_ERR_BAD_ARG;
    for (int k = 0; k < K; ++k) set_status(st + k, KA_OK);
    if (!c) return fail_members(st, K, KA_ERR_NO_DEVICE);
    if (K > KA_MAX_CANDIDATES || out_stride > 3) return fail_members(st, K, KA_ERR_LIMIT);
    if (out_stride < 1) return fail_members(st, K, KA_ERR_BAD_ARG);
    return KA_OK;
}

// What ka_ctx_set_brokers refuses in any of the K broker tables of a batched solve (the same code).
int check_tables(int K, const int32_t* cand_off, const int32_t* broker_id, const int32_t* broker_rack) {
    if (!cand_off || cand_off[0] != 0) return KA_ERR_BAD_ARG;
    for (int k = 0; k < K; ++k) {
        const int n = cand_off[k + 1] - cand_off[k];
        if (cand_off[k + 1] < cand_off[k] || (n > 0 && (!broker_id || !broker_rack))) return KA_ERR_BAD_ARG;
        const int rc = n > 0 ? check_brokers(n, broker_id + cand_off[k], broker_rack + cand_off[k]) : KA_OK;
        if (rc != KA_OK) return rc;
    }
    return KA_OK;
}

// Where one member of a batched solve reads and writes (the host side of its KaCandidate), and what its table and its slice
// need of the call's plan: a candidate table over the whole input, or one cluster of a fleet.
struct BatchMember {
    int tab = 0;                 // its broker table cand_off[tab] .. cand_off[tab + 1] - 1, and its status st[tab]
    int t0 = 0, T = 0;           // its topics [t0, t0 + T) of the shared input
    int64_t row0 = 0, Q = 0;     // its rows [row0, row0 + Q) of the shared input
    int desired_rf = -1;
    int64_t rec0 = 0;            // its first record in the call's records = its first position in the call-wide chunk table
    int64_t topic0 = 0;          // its first topic in the call's topic tables (ntl, loff, status)
    int n = 0, blob_bytes = 0;   // its table's brokers and blob
    int Pmax = 0;                // its largest topic
    int64_t capmax = 0;          // its largest capacity under its table (dense_capmax / ragged_capmax)
    int S = 1;                   // a fleet cluster's row width, which its own plan is checked with
};

// A batched solve: its K broker tables, its members and the call-wide sizes that follow from them.
struct Batch {
    int K = 0;                   // the call's K (reported by ka_ctx_last_*_plan; a fleet's refused clusters are no member)
    const int32_t* cand_off = nullptr;   // table k: broker_id[cand_off[k] .. cand_off[k + 1]) of the call
    const int32_t* broker_id = nullptr;
    std::vector<BrokerTable> tabs;       // their device images
    std::vector<BatchMember> m;
    int64_t recs = 0;            // records of the call, laid out as its output rows: K·Q for candidates, ΣP for a fleet
    int topics = 0;              // topics of the call's topic tables: K·T for candidates, ΣT for a fleet
    int fill_T = 0;              // ka_level_fill_kernel's view: topic u starts at record (u / fill_T)·fill_rows + part_off[u % fill_T]
    int64_t fill_rows = 0;
    int64_t out_rows = 0;        // output rows between two members: Q for candidates, 0 for a fleet (rows at their input rows)
    // The largest member, which the call's plan and launches are sized for: counter placement and loop shape from the largest
    // table and blob, levels and load width from the largest capacity, grids from the most topics and rows.
    int nmax = 0, blob_max = 0, Pmax = 0, Tmax = 0;
    int64_t capmax = 0, Qmax = 0;

    void add(const BatchMember& mb) {
        m.push_back(mb);
        nmax = std::max(nmax, mb.n);
        blob_max = std::max(blob_max, mb.blob_bytes);
        Pmax = std::max(Pmax, mb.Pmax);
        capmax = std::max(capmax, mb.capmax);
        Tmax = std::max(Tmax, mb.T);
        Qmax = std::max(Qmax, mb.Q);
    }
};

// The K tables of a batched call into b, once the call's own checks have passed (check_tables among them): the call's `recs`
// records (K·Q for K candidates over Q rows, ΣP for a fleet) within the 32-bit positions of the call-wide level table, the
// ctx's device, fresh plan reports, and each table's device image. A failure here fails every member.
int batch_tables(ka_ctx* c, int K, const int32_t* cand_off, const int32_t* broker_id, const int32_t* broker_rack, int64_t recs,
                 Batch& b, ka_status* st) {
    if (recs >= ((int64_t)1 << 31)) return fail_members(st, K, KA_ERR_LIMIT);
    const int rc = enter(c, true);
    if (rc != KA_OK) return fail_members(st, K, rc);
    reset_plans(c);
    b.K = K;
    b.cand_off = cand_off;
    b.broker_id = broker_id;
    b.tabs.resize(K);
    for (int k = 0; k < K; ++k)
        b.tabs[k] = broker_table(cand_off[k + 1] - cand_off[k], broker_id + cand_off[k], broker_rack + cand_off[k]);
    return KA_OK;
}

// The members of K candidates over one problem of T topics and Q rows whose largest topic has Pmax partitions, candidate k
// with the largest capacity capmax[k] under its table: every member reads the whole input, on its own copy of the records.
void add_candidates(Batch& b, int T, int64_t Q, int Pmax, int desired_rf, const std::vector<int64_t>& capmax) {
    const int64_t q = std::max<int64_t>(Q, 1);
    for (int k = 0; k < b.K; ++k)
        b.add(BatchMember{k, 0, T, 0, Q, desired_rf, (int64_t)k * q, (int64_t)k * T, b.cand_off[k + 1] - b.cand_off[k],
                          b.tabs[k].blob_bytes(), Pmax, capmax[k]});
    b.recs = (int64_t)b.K * q;
    b.topics = b.K * T;
    b.fill_T = T;
    b.fill_rows = Q;
    b.out_rows = Q;
}

// The members of a fleet of T topics over Q rows: each cluster of `passed` (those that passed ragged_scan and ragged_capmax,
// with their slice, n, Pmax, capmax and width) that also passes the limits of ka_solve's own plan under its table. A cluster
// refused there reports that limit in st[tab] and is left out, as are all clusters when none has a topic.
void add_clusters(Batch& b, int T, int64_t Q, const std::vector<BatchMember>& passed, ka_status* st) {
    for (BatchMember mb : passed) {
        mb.blob_bytes = b.tabs[mb.tab].blob_bytes();
        Plan own;
        if (make_plan(mb.n, mb.blob_bytes, mb.Q, mb.S, mb.Pmax, mb.capmax, true, own, st + mb.tab) == KA_OK) b.add(mb);
    }
    // one table of the call's T topics over its Q rows: every record sits at its input row
    b.recs = std::max<int64_t>(Q, 1);
    b.topics = T;
    b.fill_T = std::max(T, 1);
    b.out_rows = 0;
    if (b.Tmax == 0) b.m.clear();   // no topic to solve: every cluster that passed has solved (ka_solve with T == 0)
}

// The plan of a batched solve of the problem sh (one block), sized for the batch's largest member: a limit it exceeds fails
// every st[k] alike.
int plan_batch(Shape sh, const Batch& b, StageDesc& d, ka_status* st) {
    sh.Pmax = b.Pmax;
    sh.capmax = b.capmax;
    const int rc = describe_block(sh, 0, sh.T, 0, b.nmax, b.blob_max, d, st);
    for (int k = 1; k < b.K && rc != KA_OK; ++k) st[k] = st[0];
    return rc;
}

// Wait for a batched solve enqueued on `s` and fill every member's status: its lowest failing topic, as finish_status
// reports it for one solve (relative to the member's first topic; part_id / part_off of a ragged solve: the failing
// partition's id). Statuses already in st (a fleet's refused clusters) stay. Returns the code of the lowest failing st[k].
int finish_batch(ka_ctx* c, cudaStream_t s, const Batch& b, ka_status* st, const int32_t* part_id = nullptr,
                 const int64_t* part_off = nullptr) {
    const int K = b.K, M = (int)b.m.size();
    if (cudaStreamSynchronize(s) != cudaSuccess) return fail_members(st, K, KA_ERR_CUDA);
    std::vector<unsigned> err(std::max(M, 1));
    if (M > 0 && cudaMemcpy(err.data(), c->batch_run.flags.p, (size_t)M * 4, cudaMemcpyDeviceToHost) != cudaSuccess)
        return fail_members(st, K, KA_ERR_CUDA);
    for (int k = 0; k < M; ++k) {
        if (err[k] == 0xFFFFFFFFu) continue;
        const BatchMember& mb = b.m[k];
        const int t = (int)err[k] - mb.t0;   // kernel A reports the input topic
        int4 ts;
        if (cudaMemcpy(&ts, c->batch_run.tstatus.as<int4>() + mb.topic0 + t, sizeof(int4), cudaMemcpyDeviceToHost) != cudaSuccess)
            return fail_members(st, K, KA_ERR_CUDA);
        st[mb.tab] = topic_status(mb.t0 + t, ts, part_id, part_off);
        st[mb.tab].topic_index = t;
    }
    for (int k = 0; k < K; ++k)
        if (st[k].code != KA_OK) return st[k].code;
    return KA_OK;
}

// The two peak kernels over a bucket log of n buckets of indices below N, into the fields F names of sum[W].
template <typename F>
void enq_wave_peaks(ka_ctx* c, cudaStream_t s, const KaWaveBucket* log, unsigned n, int N, typename F::S* sum) {
    const unsigned blocks = (unsigned)std::max<int64_t>(1, std::min<int64_t>(((int64_t)n + 255) / 256, (int64_t)c->sm_count * 8));
    ka_wave_peak_kernel<false, F><<<blocks, 256, 0, s>>>(log, n, N, sum);
    ka_wave_peak_kernel<true, F><<<blocks, 256, 0, s>>>(log, n, N, sum);
    c->launches += 2;
}

}  // namespace

// =================================================================================================
extern "C" {

const char* ka_version(void) { return "kassign-b200 0.1 (sm_90a)"; }

int32_t ka_java_string_hash(const char* s) {
    // java.lang.String.hashCode over UTF-16 code units (KAS:190)
    uint32_t h = 0;
    const unsigned char* u = reinterpret_cast<const unsigned char*>(s);
    while (*u) {
        uint32_t cp;
        int extra;
        unsigned char b = *u++;
        if (b < 0x80) { cp = b; extra = 0; }
        else if ((b & 0xE0) == 0xC0) { cp = b & 0x1F; extra = 1; }
        else if ((b & 0xF0) == 0xE0) { cp = b & 0x0F; extra = 2; }
        else if ((b & 0xF8) == 0xF0) { cp = b & 0x07; extra = 3; }
        else { cp = 0xFFFD; extra = 0; }
        while (extra-- > 0 && *u) cp = (cp << 6) | (*u++ & 0x3F);
        if (cp >= 0x10000) {
            cp -= 0x10000;
            h = h * 31u + (0xD800u + (cp >> 10));
            h = h * 31u + (0xDC00u + (cp & 0x3FFu));
        } else {
            h = h * 31u + cp;
        }
    }
    return (int32_t)h;
}

// The bytes at which a character ka_json_name_refused refuses can start: one table lookup per byte of a name that passes.
struct NameStops {
    bool at[256];
    constexpr NameStops() : at() {
        for (int b = 0; b < 0x20; ++b) at[b] = true;
        at[(int)'"'] = at[(int)'\\'] = at[(int)'/'] = at[0xC2] = at[0xE2] = true;
    }
};
static constexpr NameStops kNameStops{};

int32_t ka_json_name_refused(const char* name, int64_t len) {
    // org.json 20131018 JSONObject.quote rewrites ", \, "</", chars below 0x20 and those in [0x80, 0xA0) and [0x2000, 0x2100);
    // the device emitter copies names verbatim, so it refuses all of them, and every '/'
    const unsigned char* u = reinterpret_cast<const unsigned char*>(name);
    for (int64_t i = 0; i < len; ++i) {
        const unsigned char b = u[i];
        if (!kNameStops.at[b]) continue;
        if (b < 0x20 || b == '"' || b == '\\' || b == '/') return b;
        if (b == 0xC2 && i + 1 < len && u[i + 1] >= 0x80 && u[i + 1] < 0xA0) return u[i + 1];   // U+0080..U+009F
        if (b == 0xE2 && i + 2 < len && u[i + 1] >= 0x80 && u[i + 1] < 0x84 && (u[i + 2] & 0xC0) == 0x80)
            return 0x2000 | ((u[i + 1] & 0x3F) << 6) | (u[i + 2] & 0x3F);                     // U+2000..U+20FF
    }
    return -1;
}

int32_t ka_rack_indices(int32_t N, const int32_t* broker_id, const char* const* rack_name, int32_t* broker_rack) {
    if (N < 0 || (N > 0 && (!broker_id || !broker_rack))) return KA_ERR_BAD_ARG;
    // rack key = the rack string, or Integer.toString(id) when no rack is defined (KAS:81-86); brokers
    // share a Rack object iff their keys are equal strings (KAS:90-94).
    std::map<std::string, int32_t> key2idx;
    for (int i = 0; i < N; ++i) {
        std::string key = (rack_name && rack_name[i]) ? std::string(rack_name[i]) : std::to_string(broker_id[i]);
        auto it = key2idx.find(key);
        if (it == key2idx.end()) it = key2idx.emplace(key, (int32_t)key2idx.size()).first;
        broker_rack[i] = it->second;
    }
    return KA_OK;
}

ka_ctx* ka_ctx_create(int32_t device) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
        cudaGetLastError();
        return nullptr;
    }
    if (cudaSetDevice(device) != cudaSuccess) return nullptr;
    ka_ctx* c = new (std::nothrow) ka_ctx();
    if (!c) return nullptr;
    c->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) c->sm_count = prop.multiProcessorCount;
    bool ok = cudaHostAlloc(reinterpret_cast<void**>(&c->h_pin), sizeof(HostPinned), cudaHostAllocDefault) == cudaSuccess &&
              cudaHostAlloc(reinterpret_cast<void**>(&c->h_frag), 2 * KA_MAX_JSON_FRAGS * sizeof(unsigned long long),
                            cudaHostAllocDefault) == cudaSuccess;
    for (cudaStream_t* s : c->streams())
        ok = ok && cudaStreamCreateWithFlags(s, cudaStreamNonBlocking) == cudaSuccess;
    for_each_event(c, [&](cudaEvent_t& e, bool timed) {
        ok = ok && cudaEventCreateWithFlags(&e, timed ? cudaEventDefault : cudaEventDisableTiming) == cudaSuccess;
    });
    if (!ok) {   // release whatever was created
        ka_ctx_destroy(c);
        return nullptr;
    }
    return c;
}

void ka_ctx_destroy(ka_ctx* c) {
    if (!c) return;
    enter_host(c);   // a pending asynchronous call still uses the buffers on the caller's stream: wait for it first
    for (cudaStream_t* s : c->streams())
        if (*s) cudaStreamSynchronize(*s);
    for_each_event(c, [](cudaEvent_t& e, bool) { if (e) cudaEventDestroy(e); });
    for (cudaStream_t* s : c->streams())
        if (*s) cudaStreamDestroy(*s);
    if (c->h_pin) cudaFreeHost(c->h_pin);
    if (c->h_frag) cudaFreeHost(c->h_frag);
    delete c;   // the DevBufs free themselves, on c->device
}

int32_t ka_ctx_reset(ka_ctx* c) {
    if (!c) return KA_ERR_NO_DEVICE;
    int rc = enter_host(c);   // do not race an in-flight asynchronous call
    if (rc != KA_OK) return rc;
    c->parked.clear();
    if (c->br.N > 0 && c->d_ctr8.p) KA_CUDA(cudaMemset(c->d_ctr8.p, 0, (size_t)c->br.N * KA_MAX_SLOTS * 4));
    return KA_OK;
}

int32_t ka_ctx_set_brokers(ka_ctx* c, int32_t N, const int32_t* broker_id, const int32_t* broker_rack) {
    if (!c) return KA_ERR_NO_DEVICE;
    int rc = check_brokers(N, broker_id, broker_rack);
    if (rc != KA_OK) return rc;
    if ((rc = enter_host(c)) != KA_OK || (rc = park_counters(c)) != KA_OK) return rc;

    const BrokerTable t = broker_table(N, broker_id, broker_rack);
    if (t.lut_mode == KA_LUT_GLOBAL) {
        KA_CUDA(c->d_glut.reserve(t.glut.size() * 2));
        KA_CUDA(cudaMemcpy(c->d_glut.p, t.glut.data(), t.glut.size() * 2, cudaMemcpyHostToDevice));
    }
    KA_CUDA(c->d_blob.reserve(t.blob.size() * 2));
    KA_CUDA(cudaMemcpy(c->d_blob.p, t.blob.data(), t.blob.size() * 2, cudaMemcpyHostToDevice));
    KA_CUDA(c->d_broker_id.reserve((size_t)std::max(N, 1) * 4));
    if (N > 0) KA_CUDA(cudaMemcpy(c->d_broker_id.p, broker_id, (size_t)N * 4, cudaMemcpyHostToDevice));
    c->br = t.device(N, c->d_blob.as<uint16_t>(), c->d_glut.as<uint16_t>(), c->d_broker_id.as<int32_t>());
    c->broker_id.assign(broker_id, broker_id + N);
    // counters for the new table
    std::vector<int32_t> h((size_t)(std::max(N, 1) + 1) * KA_MAX_SLOTS, 0);  // + the order kernel's dummy row (index N)
    for (int i = 0; i < N; ++i) {
        auto it = c->parked.find(broker_id[i]);
        if (it != c->parked.end()) std::copy(it->second.begin(), it->second.end(), h.begin() + (size_t)i * KA_MAX_SLOTS);
    }
    KA_CUDA(c->d_ctr8.reserve(h.size() * 4));
    KA_CUDA(cudaMemcpy(c->d_ctr8.p, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
    return KA_OK;
}

int32_t ka_ctx_counter_slots(ka_ctx*) { return KA_MAX_SLOTS; }

int32_t ka_ctx_get_counters(ka_ctx* c, int32_t* counter) {
    if (!c) return KA_ERR_NO_DEVICE;
    if (!counter) return KA_ERR_BAD_ARG;
    int rc = enter_host(c);
    if (rc != KA_OK) return rc;
    if (c->br.N > 0) KA_CUDA(cudaMemcpy(counter, c->d_ctr8.p, (size_t)c->br.N * KA_MAX_SLOTS * 4, cudaMemcpyDeviceToHost));
    return KA_OK;
}

int32_t ka_ctx_set_counters(ka_ctx* c, const int32_t* counter) {
    if (!c) return KA_ERR_NO_DEVICE;
    if (!counter) return KA_ERR_BAD_ARG;
    int rc = enter_host(c);
    if (rc != KA_OK) return rc;
    if (c->br.N > 0) KA_CUDA(cudaMemcpy(c->d_ctr8.p, counter, (size_t)c->br.N * KA_MAX_SLOTS * 4, cudaMemcpyHostToDevice));
    return KA_OK;
}

int32_t ka_ctx_export_counters_device(ka_ctx* c, int32_t* d_counter, void* stream) {
    if (!c) return KA_ERR_NO_DEVICE;
    if (!d_counter) return KA_ERR_BAD_ARG;
    int rc = enter(c, false);
    if (rc != KA_OK) return rc;
    if (c->br.N > 0)
        KA_CUDA(cudaMemcpyAsync(d_counter, c->d_ctr8.p, (size_t)c->br.N * KA_MAX_SLOTS * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return end_untracked(c, (cudaStream_t)stream);
}

int32_t ka_ctx_import_counters_device(ka_ctx* c, const int32_t* d_counter, void* stream) {
    if (!c) return KA_ERR_NO_DEVICE;
    if (!d_counter) return KA_ERR_BAD_ARG;
    int rc = enter(c, false);
    if (rc != KA_OK) return rc;
    if (c->br.N > 0)
        KA_CUDA(cudaMemcpyAsync(c->d_ctr8.p, d_counter, (size_t)c->br.N * KA_MAX_SLOTS * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return end_untracked(c, (cudaStream_t)stream);
}

int32_t ka_ctx_set_timing(ka_ctx* c, int32_t enabled) {
    if (!c) return KA_ERR_NO_DEVICE;
    c->timing = enabled != 0;
    return KA_OK;
}

int32_t ka_ctx_set_wave_rule(ka_ctx* c, int32_t rule) {
    if (!c) return KA_ERR_NO_DEVICE;
    if (rule != KA_WAVE_GREEDY && rule != KA_WAVE_FIRST_FIT) return KA_ERR_BAD_ARG;
    c->wave_rule = rule;
    return KA_OK;
}

int32_t ka_ctx_wave_rule(ka_ctx* c) { return c ? c->wave_rule : KA_ERR_NO_DEVICE; }

int32_t ka_ctx_set_part_caps(ka_ctx* c, int64_t max_part_rows, int64_t max_part_in) {
    if (!c) return KA_ERR_NO_DEVICE;
    if (max_part_rows < 0 || max_part_in < 0) return KA_ERR_BAD_ARG;
    c->part_rows = max_part_rows;
    c->part_in = max_part_in;
    return KA_OK;
}

int32_t ka_ctx_part_caps(ka_ctx* c, int64_t* max_part_rows, int64_t* max_part_in) {
    if (!c) return KA_ERR_NO_DEVICE;
    if (!max_part_rows || !max_part_in) return KA_ERR_BAD_ARG;
    *max_part_rows = c->part_rows;
    *max_part_in = c->part_in;
    return KA_OK;
}

int32_t ka_ctx_last_timing(ka_ctx* c, float* ms) {
    if (!c) return KA_ERR_NO_DEVICE;
    if (!ms) return KA_ERR_BAD_ARG;
    for (int i = 0; i < 8; ++i) ms[i] = c->last_ms[i];
    return KA_OK;
}

int64_t ka_ctx_launch_count(ka_ctx* c) { return c ? c->launches : 0; }

int32_t ka_ctx_last_order_plan(ka_ctx* c, int32_t* plan) {
    if (!c || !plan) return KA_ERR_BAD_ARG;
    for (int i = 0; i < 8; ++i) plan[i] = c->order_plan[i];
    return KA_OK;
}

int32_t ka_ctx_last_stage_plan(ka_ctx* c, int32_t* plan) {
    if (!c || !plan) return KA_ERR_BAD_ARG;
    for (int i = 0; i < 8; ++i) plan[i] = c->stage_plan[i];
    return KA_OK;
}

int32_t ka_last_status(ka_ctx* c, ka_status* st) {
    if (!c) return set_status(st, KA_ERR_NO_DEVICE);
    int rc = enter(c, false);
    if (rc != KA_OK || (rc = wait_untracked(c)) != KA_OK) return set_status(st, rc);
    if (c->pending_status) return finish_status(c, c->last_stream, st);
    if (st) *st = c->last;
    return c->last.code;
}

static int validate_dense(ka_ctx* c, int32_t T, int32_t P, int32_t RF, int32_t desired_rf, int32_t S, ka_status* st) {
    set_status(st, KA_OK);
    if (!c) return set_status(st, KA_ERR_NO_DEVICE);
    if (T < 0 || P < 0 || RF < 0) return set_status(st, KA_ERR_BAD_ARG);
    if (S < 1 || S > KA_MAX_SLOTS) return set_status(st, KA_ERR_LIMIT, -1, -1, S);
    const int rf_t = desired_rf >= 0 ? desired_rf : RF;
    if (S < RF || (rf_t <= c->br.N && S < rf_t)) return set_status(st, KA_ERR_BAD_ARG, -1, -1, S);
    return KA_OK;
}

int32_t ka_solve_dense_device(ka_ctx* c, int32_t T, const int32_t* d_topic_hash, int32_t P, int32_t RF,
                              const int32_t* d_cur_broker, int32_t desired_rf, int32_t out_stride,
                              int32_t* d_out_len, int32_t* d_out_broker, void* stream, ka_status* st) {
    int rc = validate_dense(c, T, P, RF, desired_rf, out_stride, st);
    if (rc != KA_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    SolveCall io(d_out_broker, d_out_len);
    const Shape sh = dense_shape(T, P, RF, desired_rf, out_stride, c->br.N, d_topic_hash, d_cur_broker);
    if ((rc = enter(c, true)) != KA_OK || (rc = run_solve(c, s, sh, io, st)) != KA_OK) return failed(st, rc);
    return finish(c, s, st, false);
}

// Everything of a batched solve over the members of `bt`, enqueued on `s` (slot-0 chains on c->sb1): the members' tables
// and descriptors H2D, fresh counters, kernel A with grid.y = member, the level tables of all members as one table, then per
// chain sub-block the slot-0 / slot-1 chains (one CTA per member) and the emit (grid.y = member). `d` is a dense problem or a
// ragged one (d.d_part_off set: one chain sub-block, as in a ragged single solve); its inputs are shared by every member, each
// of which reads its own window of them.
static int enq_batch(ka_ctx* c, cudaStream_t s, const Batch& bt, const StageDesc& d, int32_t* d_out_len, int32_t* d_out) {
    const Plan& pl = d.pl;
    const int S = d.S, K = (int)bt.m.size();
    const size_t kq = (size_t)bt.recs, kt = (size_t)bt.topics;
    // the members' tables, in one upload: the descriptors (first: score_batch reads them at d_batch_tab), then every member's
    // blob, global LUT and broker ids
    struct MemberTab { uint16_t *blob, *glut; int32_t* bid; };
    struct Tables { KaCandidate* cand; std::vector<MemberTab> m; };
    const auto tables = [&](Layout& l) {
        Tables o{l.take<KaCandidate>(K), {}};
        for (const BatchMember& mb : bt.m)
            o.m.push_back({l.take<uint16_t>(bt.tabs[mb.tab].blob.size()), l.take<uint16_t>(bt.tabs[mb.tab].glut.size()),
                           l.take<int32_t>(std::max(mb.n, 1))});
        return o;
    };
    const auto counters = [&](Layout& l) {   // every member's counters, + the chains' dummy row
        std::vector<int32_t*> ctr8;
        for (const BatchMember& mb : bt.m) ctr8.push_back(l.take<int32_t>((size_t)(mb.n + 1) * KA_MAX_SLOTS));
        return ctr8;
    };
    std::vector<unsigned char> h(layout_bytes(tables), 0);
    const size_t ctr_bytes = layout_bytes(counters);
    RunScratch& r = c->batch_run;
    KA_CUDA(c->d_batch_tab.reserve(h.size()));
    KA_CUDA(c->d_batch_ctr.reserve(ctr_bytes));
    KA_CUDA(r.reserve(kq * 16, kq, kt, kt + 1, pl.a_levels, K));
    const Tables host = place(tables, h.data()), dev = place(tables, c->d_batch_tab.p);
    const std::vector<int32_t*> ctr8 = place(counters, c->d_batch_ctr.p);
    int lut_mask = 0;
    int64_t covered = 0;   // topics kernel A walks
    for (int k = 0; k < K; ++k) {
        const BatchMember& mb = bt.m[k];
        const BrokerTable& t = bt.tabs[mb.tab];
        // kernel A writes the member's records, perm and lend by input row, its ntl and status by input topic
        const int64_t shift = mb.rec0 - mb.row0, tshift = mb.topic0 - mb.t0;
        KaCandidate e{};
        e.br = t.device(mb.n, dev.m[k].blob, dev.m[k].glut, dev.m[k].bid);
        e.ctr8 = ctr8[k];
        e.out.rec = r.rec.as<unsigned char>() + shift * 16;
        if (pl.a_levels) {
            e.out.perm = r.perm.as<uint16_t>() + shift;
            e.out.ntl = r.ntl.as<int32_t>() + tshift;
            e.out.lend = r.lend.as<uint32_t>() + shift;
            e.loff = r.loff.as<int32_t>() + mb.topic0;
            e.pos0 = (uint32_t)mb.rec0;   // the level tables of the members are one table of bt.topics topics
        }
        e.out.tstatus = r.tstatus.as<int4>() + tshift;
        e.out.err_topic = r.flags.as<unsigned>() + k;
        e.desired_rf = mb.desired_rf;
        e.t0 = mb.t0;
        e.T = mb.T;
        e.row0 = (uint32_t)mb.row0;
        e.Q = (uint32_t)mb.Q;
        std::memcpy(host.cand + k, &e, sizeof(e));
        std::memcpy(host.m[k].blob, t.blob.data(), t.blob.size() * 2);
        if (!t.glut.empty()) std::memcpy(host.m[k].glut, t.glut.data(), t.glut.size() * 2);
        if (mb.n > 0) std::memcpy(host.m[k].bid, bt.broker_id + bt.cand_off[mb.tab], (size_t)mb.n * 4);
        lut_mask |= 1 << t.lut_mode;
        covered += mb.T;
    }
    const KaCandidate* cand = dev.cand;
    KA_CUDA(cudaMemcpyAsync(c->d_batch_tab.p, h.data(), h.size(), cudaMemcpyHostToDevice, s));
    KA_CUDA(cudaMemsetAsync(c->d_batch_ctr.p, 0, ctr_bytes, s));   // every member starts from a fresh Context
    KA_CUDA(cudaMemsetAsync(r.flags.p, 0xFF, (size_t)K * 4, s));
    // topics no member walks (a fleet's refused clusters) have no chunks
    if (pl.a_levels && covered < bt.topics) KA_CUDA(cudaMemsetAsync(r.ntl.p, 0, kt * 4, s));
    // kernel A: grid.y = member, grid.x from the largest member; the plan's shared-memory layout is that of the largest table
    KaSolveParams p = stage_params(d);
    p.cand = cand;
    int rc = launch_stage_plan<true>(c, s, p, pl, bt.Tmax, K, lut_mask);
    if (rc != KA_OK) return rc;
    c->stage_plan[3] = bt.K;
    if (pl.a_levels) {
        ka_level_scan_kernel<<<1, 1024, 0, s>>>(r.ntl.as<int32_t>(), (int)kt, r.loff.as<int32_t>());
        KA_CUDA(cudaGetLastError());
        ka_level_fill_kernel<<<(unsigned)((kt + 7) / 8), 256, 0, s>>>(r.ntl.as<int32_t>(), r.loff.as<int32_t>(), r.lend.as<uint32_t>(),
                                                                      d.d_part_off, d.P, bt.fill_T, (int)kt, bt.fill_rows,
                                                                      r.lvl_end.as<uint32_t>());
        KA_CUDA(cudaGetLastError());
        c->launches += 2;
    }
    if (bt.Qmax <= 0) return KA_OK;
    // the chains: slot 0 of sub-block j+1 (c->sb1) overlaps slot 1 + emit of sub-block j (s), as in the single solve. A launch
    // covers the sub-block's rows and topics; every member clips them to its own window.
    if ((rc = chain_fork(c, s)) != KA_OK) return rc;
    const int nsub = chain_subblocks(d, 1);
    for (int j = 0; j < nsub; ++j) {
        const SubBlock b = sub_block(d, j, nsub);
        KaOrderParams o{};
        o.N = 0;
        o.S = S;
        o.uniform_width = pl.a_levels ? 0u : (uint32_t)d.P;
        o.chunk_end = pl.a_levels ? r.lvl_end.as<uint32_t>() : nullptr;
        o.ring_log2 = pl.b_ring_log2;
        o.Q = (uint32_t)b.rq;
        o.pos_base = (uint32_t)b.r0;
        o.cand = cand;
        o.cand_t0 = b.t0;
        o.cand_t1 = b.t1;
        int sel = 0;
        KA_CUDA((launch_order<0, 1024, true>(c->sb1, o, pl, &sel, K)));
        note_order(c, pl, sel, bt.K);
        KA_CUDA(cudaEventRecord(c->ev_b1[j], c->sb1));
        KA_CUDA(cudaStreamWaitEvent(s, c->ev_b1[j], 0));
        KA_CUDA((launch_order<1, 1024, true>(s, o, pl, &sel, K)));
        note_order(c, pl, sel, bt.K);
        const int64_t rq = std::min(b.rq, bt.Qmax);   // the largest member's rows of the sub-block
        const dim3 grid((unsigned)((rq + 255) / 256), K);
        if (d.d_part_off)
            ka_emit3_candidates_kernel<true><<<grid, 256, 0, s>>>(cand, 0u, d.T, 0, d.d_part_off, (uint32_t)rq, S, bt.out_rows, d_out,
                                                                  d_out_len);
        else
            ka_emit3_candidates_kernel<<<grid, 256, 0, s>>>(cand, (uint32_t)b.r0, b.t1 - b.t0, d.P, nullptr, (uint32_t)rq, S, bt.out_rows,
                                                            d_out, d_out_len);
        KA_CUDA(cudaGetLastError());
        c->launches += 3;
    }
    return KA_OK;
}

// The batched solve planned as d, enqueued on `s`: the host inputs H2D when io has any (ncur current replicas), the batch, and
// the rows of every member D2H when io has a host destination. A failure after something was enqueued fails every member.
static int run_batch(ka_ctx* c, cudaStream_t s, const Batch& bt, const StageDesc& d, int64_t ncur, const SolveCall& io,
                     ka_status* st) {
    int rc;
    if ((rc = enq_inputs(s, io, d, ncur)) != KA_OK || (rc = enq_batch(c, s, bt, d, io.d_out_len, io.d_out)) != KA_OK ||
        (io.h_out && d.Q > 0 && (rc = enq_copy_out(s, io, d.S, 0, bt.recs)) != KA_OK))
        return abort_batch(c, s, st, bt.K, rc);
    return KA_OK;
}

int32_t ka_solve_dense_candidates_device(ka_ctx* c, int32_t K, const int32_t* cand_off, const int32_t* broker_id,
                                         const int32_t* broker_rack, int32_t T, const int32_t* d_topic_hash, int32_t P,
                                         int32_t RF, const int32_t* d_cur_broker, int32_t desired_rf, int32_t out_stride,
                                         int32_t* d_out_len, int32_t* d_out_broker, void* stream, ka_status* st) {
    int rc = batch_args(c, K, out_stride, st);
    if (rc != KA_OK) return rc;
    if (T < 0 || P < 0 || RF < 0 || out_stride < std::max(RF, desired_rf)) return fail_members(st, K, KA_ERR_BAD_ARG);
    if (K == 0) return KA_OK;
    if ((rc = check_tables(K, cand_off, broker_id, broker_rack)) != KA_OK) return fail_members(st, K, rc);
    if (T == 0) return KA_OK;
    const int64_t Q = (int64_t)T * P;
    if (!d_topic_hash || (Q * RF > 0 && !d_cur_broker) || (Q > 0 && !d_out_broker)) return fail_members(st, K, KA_ERR_BAD_ARG);
    Batch bt;
    if ((rc = batch_tables(c, K, cand_off, broker_id, broker_rack, (int64_t)K * Q, bt, st)) != KA_OK) return rc;
    // levels if any candidate that can serve the target RF has capacity > 1 (one that cannot fails alone, whatever the plan)
    const int rf_t = desired_rf >= 0 ? desired_rf : RF;
    std::vector<int64_t> cap(K);
    for (int k = 0; k < K; ++k) cap[k] = dense_capmax(P, rf_t, cand_off[k + 1] - cand_off[k]);
    add_candidates(bt, T, Q, P, desired_rf, cap);
    const Shape sh = dense_shape(T, P, RF, desired_rf, out_stride, 0, d_topic_hash, d_cur_broker);   // sized by plan_batch
    const SolveCall io(d_out_broker, d_out_len);
    cudaStream_t s = (cudaStream_t)stream;
    StageDesc d;
    if ((rc = plan_batch(sh, bt, d, st)) != KA_OK || (rc = run_batch(c, s, bt, d, 0, io, st)) != KA_OK) return rc;
    return finish_batch(c, s, bt, st);
}

int32_t ka_stage_dense_device(ka_ctx* c, int32_t T, const int32_t* d_topic_hash, int32_t P, int32_t RF,
                              const int32_t* d_cur_broker, int32_t desired_rf, int32_t out_stride, void* stream) {
    ka_status lst;
    int rc = validate_dense(c, T, P, RF, desired_rf, out_stride, &lst);
    if (rc != KA_OK || (rc = enter(c, true)) != KA_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    StageDesc& d = c->staged_block;
    c->staged = false;
    reset_plans(c);
    const Shape sh = dense_shape(T, P, RF, desired_rf, out_stride, c->br.N, d_topic_hash, d_cur_broker);
    if ((rc = describe_block(sh, 0, T, 0, c->br.N, c->br.blob_bytes, d, &lst)) != KA_OK ||
        (rc = reserve_scratch(c, &d, 1)) != KA_OK)
        return rc;
    c->last_stages = 1;
    if (c->timing) { cudaEventRecord(c->ev[0], s); cudaEventRecord(c->ev[1], s); }
    if ((rc = reset_flags(c, s)) != KA_OK || (rc = enq_stage(c, s, d, c->ev[2])) != KA_OK) return rc;
    if (c->timing) cudaEventRecord(c->ev[3], s);   // end of the stage (the chains may wait for another rank after this)
    c->staged = true;
    return end_untracked(c, s);
}

// Prologue of the calls that finish the staged block: st cleared, the ctx, its device made current, then a staged block
// (with slot_chains, one whose leader order is the two slot chains of rows <= 3); the first that fails is reported.
static int enter_staged(ka_ctx* c, bool slot_chains, ka_status* st) {
    set_status(st, KA_OK);
    if (!c) return set_status(st, KA_ERR_NO_DEVICE);
    const int rc = enter(c, false);
    if (rc != KA_OK) return failed(st, rc);
    if (!c->staged || (slot_chains && c->staged_block.pl.rec_kind != 3)) return set_status(st, KA_ERR_BAD_ARG);
    return KA_OK;
}

// End of the staged block's solve, its rows enqueued on `s`: the block is used up and its status pending on `s`.
static int end_staged(ka_ctx* c, cudaStream_t s, ka_status* st) {
    if (c->timing) cudaEventRecord(c->ev[4], s);
    const int rc = enq_solve_end(c, s);
    if (rc != KA_OK) return failed(st, rc);
    c->staged = false;
    c->last_was_staged = true;
    return finish(c, s, st, false);
}

int32_t ka_order_device(ka_ctx* c, int32_t* d_out_len, int32_t* d_out_broker, void* stream, ka_status* st) {
    int rc = enter_staged(c, false, st);
    if (rc != KA_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    SolveCall io(d_out_broker, d_out_len);
    if ((rc = chain_fork(c, s)) != KA_OK || (rc = enq_order_emit(c, s, c->staged_block, io, 1)) != KA_OK ||
        (rc = join_emits(c, s, io)) != KA_OK)
        return failed(st, rc);
    return end_staged(c, s, st);
}

int32_t ka_staged_slot_chains(ka_ctx* c) {
    if (!c || !c->staged) return 0;
    return c->staged_block.pl.rec_kind == 3 ? 2 : 0;
}

int32_t ka_order_slot_device(ka_ctx* c, int32_t slot, void* stream) {
    int rc = enter_staged(c, true, nullptr);
    if (rc != KA_OK) return rc;
    if (slot < 0 || slot > 1) return KA_ERR_BAD_ARG;
    const StageDesc& d = c->staged_block;
    cudaStream_t s = (cudaStream_t)stream;
    const int nsub = chain_subblocks(d, 1);
    if (c->timing) cudaEventRecord(c->ev_chain[slot][0], s);
    for (int j = 0; j < nsub; ++j)
        if ((rc = enq_slot_chain(c, s, d, slot, j, nsub)) != KA_OK) return rc;
    if (c->timing) cudaEventRecord(c->ev_chain[slot][1], s);
    c->slot_timed[slot] = c->timing;
    return end_untracked(c, s);
}

int32_t ka_emit_device(ka_ctx* c, int32_t* d_out_len, int32_t* d_out_broker, void* stream, ka_status* st) {
    int rc = enter_staged(c, true, st);
    if (rc != KA_OK) return rc;
    if (!d_out_broker && c->staged_block.Q > 0) return set_status(st, KA_ERR_BAD_ARG);   // a block without rows writes none
    cudaStream_t s = (cudaStream_t)stream;
    if ((rc = enq_emit_block(c, s, c->staged_block, 0, 1, d_out_broker, d_out_len)) != KA_OK) return failed(st, rc);
    return end_staged(c, s, st);
}

static int copy_counter_column(ka_ctx* c, int slot, int32_t* d_col, const int32_t* d_src, cudaStream_t s) {
    if (!c) return KA_ERR_NO_DEVICE;
    if (slot < 0 || slot >= KA_MAX_SLOTS || (!d_col && !d_src)) return KA_ERR_BAD_ARG;
    int rc = enter(c, false);
    if (rc != KA_OK) return rc;
    if (c->br.N <= 0) return KA_OK;
    int32_t* col = c->d_ctr8.as<int32_t>() + slot;
    if (d_col) KA_CUDA(cudaMemcpy2DAsync(d_col, 4, col, KA_MAX_SLOTS * 4, 4, (size_t)c->br.N, cudaMemcpyDeviceToDevice, s));
    else KA_CUDA(cudaMemcpy2DAsync(col, KA_MAX_SLOTS * 4, d_src, 4, 4, (size_t)c->br.N, cudaMemcpyDeviceToDevice, s));
    return end_untracked(c, s);
}

int32_t ka_ctx_export_counter_slot_device(ka_ctx* c, int32_t slot, int32_t* d_column, void* stream) {
    return copy_counter_column(c, slot, d_column, nullptr, (cudaStream_t)stream);
}

int32_t ka_ctx_import_counter_slot_device(ka_ctx* c, int32_t slot, const int32_t* d_column, void* stream) {
    return copy_counter_column(c, slot, nullptr, d_column, (cudaStream_t)stream);
}

int32_t ka_ctx_set_topic_base(ka_ctx* c, int32_t topic_base) {
    if (!c) return KA_ERR_NO_DEVICE;
    if (topic_base < 0) return KA_ERR_BAD_ARG;
    c->topic_base = topic_base;
    return KA_OK;
}

int32_t ka_solve_dense(ka_ctx* c, int32_t T, const int32_t* topic_hash, int32_t P, int32_t RF,
                       const int32_t* cur_broker, int32_t desired_rf, int32_t out_stride,
                       int32_t* out_len, int32_t* out_broker, ka_status* st) {
    int rc = validate_dense(c, T, P, RF, desired_rf, out_stride, st);
    if (rc != KA_OK) return rc;
    if ((rc = enter_host(c)) != KA_OK) return failed(st, rc);
    Shape sh = dense_shape(T, P, RF, desired_rf, out_stride, c->br.N);
    if ((T > 0 && !topic_hash) || (sh.R > 0 && !cur_broker) || (sh.Q > 0 && !out_broker)) return set_status(st, KA_ERR_BAD_ARG);
    if ((rc = reserve_io(c, sh, false)) != KA_OK) return failed(st, rc);
    SolveCall io = host_call(c, topic_hash, nullptr, nullptr, cur_broker, out_len, out_broker);
    if ((rc = run_solve(c, c->stream, sh, io, st)) != KA_OK) return failed(st, rc);
    return finish(c, c->stream, st, true);
}

// The name slab of a text pass over T topics and Q rows H2D on s: names and name_off, and the rows' partition ids when given.
static int upload_names(ka_ctx* c, cudaStream_t s, int32_t T, int64_t Q, const char* names, const int64_t* name_off,
                        const int32_t* part_id) {
    const int64_t name_bytes = T > 0 ? name_off[T] : 0;
    KA_CUDA(c->d_names.reserve((size_t)std::max<int64_t>(name_bytes, 1)));
    KA_CUDA(c->d_name_off.reserve((size_t)(T + 1) * 8));
    if (part_id) KA_CUDA(c->d_part_id.reserve((size_t)Q * 4));
    if (name_bytes > 0) KA_CUDA(cudaMemcpyAsync(c->d_names.p, names, (size_t)name_bytes, cudaMemcpyHostToDevice, s));
    if (T > 0) KA_CUDA(cudaMemcpyAsync(c->d_name_off.p, name_off, (size_t)(T + 1) * 8, cudaMemcpyHostToDevice, s));
    if (part_id && Q > 0) KA_CUDA(cudaMemcpyAsync(c->d_part_id.p, part_id, (size_t)Q * 4, cudaMemcpyHostToDevice, s));
    return KA_OK;
}

// Device buffers of a JSON solve, and its topic names H2D (on c->sj, ahead of the first fragment; the solve uploads the
// partition ids).
static int prepare_json(ka_ctx* c, int32_t T, int64_t Q, const char* names, const int64_t* name_off, int64_t json_cap) {
    KA_CUDA(c->d_json.reserve((size_t)json_cap));
    KA_CUDA(c->d_json_rowlen.reserve((size_t)std::max<int64_t>(Q, 1) * 4));
    KA_CUDA(c->d_json_blocksum.reserve((size_t)(Q / 256 + 2 * KA_MAX_JSON_FRAGS) * 4));
    KA_CUDA(c->d_json_state.reserve((2 + 2 * KA_MAX_JSON_FRAGS) * 8));
    const int rc = upload_names(c, c->sj, T, Q, names, name_off, nullptr);
    if (rc != KA_OK) return rc;
    KA_CUDA(cudaMemsetAsync(c->d_json_state.p, 0, (2 + 2 * KA_MAX_JSON_FRAGS) * 8, c->sj));
    return KA_OK;
}

// The device emitter copies topic names verbatim: a name with a character ka_json_name_refused refuses is refused
// (KA_ERR_BAD_ARG, a = that character's code point), and the caller takes the host emitter instead. Checks the names of
// topics [t0, t1), each on its own.
static int check_names(const char* names, const int64_t* name_off, int t0, int t1, ka_status* st) {
    for (int t = t0; t < t1; ++t) {
        const int32_t cp = ka_json_name_refused(names + name_off[t], name_off[t + 1] - name_off[t]);
        if (cp >= 0) return set_status(st, KA_ERR_BAD_ARG, -1, -1, cp);
    }
    return KA_OK;
}

// A JSON solve of sh on c->stream, from the host inputs of io (no host rows), once its ctx's device copies are reserved:
// prepare_json, then the run (refused with KA_ERR_BAD_ARG when not `runnable`). Every fragment is enqueued on c->sj: stream
// each one into `json` as soon as its size is known (later fragments may still be in the chains or being built), then
// collect the solve's status (the failing partition's id when io has part ids). On any error *json_bytes stays 0; a text
// longer than json_cap is KA_ERR_LIMIT.
static int solve_json(ka_ctx* c, const Shape& sh, SolveCall io, const char* names, const int64_t* name_off, char* json,
                      int64_t json_cap, int64_t* json_bytes, ka_status* st, bool runnable = true) {
    int rc = prepare_json(c, sh.T, sh.Q, names, name_off, json_cap);
    if (rc != KA_OK) return failed(st, rc);
    cudaStream_t s = c->stream;
    io.json = true;
    if ((rc = runnable ? run_solve(c, s, sh, io, st) : KA_ERR_BAD_ARG) != KA_OK) {
        cudaStreamSynchronize(c->sj);
        return failed(st, rc);
    }
    finish(c, s, nullptr, false);   // pending: collected below, once the fragments are out
    int64_t total = 0;
    bool overflow = false;
    for (int k = 0; k < io.json_blocks; ++k) {
        KA_CUDA(cudaEventSynchronize(c->ev_json_scan[k]));
        const int64_t base = (int64_t)c->h_frag[2 * k], size = (int64_t)c->h_frag[2 * k + 1];
        if (base + size > json_cap) { overflow = true; break; }
        if (size > 0) KA_CUDA(cudaMemcpyAsync(json + base, c->d_json.as<char>() + base, (size_t)size, cudaMemcpyDeviceToHost, c->sj));
        total = base + size;
    }
    KA_CUDA(cudaStreamSynchronize(c->sj));
    rc = finish_status(c, s, st, io.h_part_id, io.h_part_off);
    if (rc == KA_OK && overflow) return set_status(st, KA_ERR_LIMIT, -1, -1, (int)std::min<int64_t>(json_cap, INT_MAX));
    if (json_bytes) *json_bytes = rc == KA_OK ? total : 0;
    return rc;
}

int32_t ka_solve_dense_json(ka_ctx* c, int32_t T, const int32_t* topic_hash, int32_t P, int32_t RF, const int32_t* cur_broker,
                            int32_t desired_rf, const char* names, const int64_t* name_off, char* json, int64_t json_cap,
                            int64_t* json_bytes, ka_status* st) {
    const int S = std::max(std::max(RF, desired_rf), 1);
    if (json_bytes) *json_bytes = 0;
    int rc = validate_dense(c, T, P, RF, desired_rf, S, st);
    if (rc != KA_OK) return rc;
    Shape sh = dense_shape(T, P, RF, desired_rf, S, c->br.N);
    if ((T > 0 && (!topic_hash || !names || !name_off)) || (sh.R > 0 && !cur_broker) || !json || json_cap < KA_JSON_HEAD_LEN + KA_JSON_TAIL_LEN)
        return set_status(st, KA_ERR_BAD_ARG);
    if ((rc = check_names(names, name_off, 0, T, st)) != KA_OK) return rc;
    if ((rc = enter_host(c)) != KA_OK || (rc = reserve_io(c, sh, false)) != KA_OK) return failed(st, rc);
    // no topics or no brokers: no text to write, refused once its buffers are prepared
    return solve_json(c, sh, host_call(c, topic_hash, nullptr, nullptr, cur_broker, nullptr, nullptr), names, name_off, json, json_cap,
                      json_bytes, st, T > 0 && c->br.N > 0);
}

// Host-side sizing scan of a ragged problem that does not depend on any broker table: offsets, list sizes, the largest
// topic, and per target RF the largest topic of that RF (the capacity bound of KAS:65-71 for any table follows from those:
// ragged_capmax). pick_max > 0: S is chosen here, as max(longest current list, desired_rf, 1), and a width above pick_max is
// KA_ERR_LIMIT (a = the width); pick_max == 0: S is the caller's. have_out: the caller has
// somewhere to put the rows. Failures that come before the topic loop are returned; those of the topic and list-size
// loops are kept in `err` (in the order ka_solve reports them), because a failure that depends on the table — a topic
// whose target RF exceeds S but not N — takes precedence when it comes from an earlier topic.
struct RaggedScan {
    int64_t Q = 0, R = 0, maxsz = 0;
    int S = 1, Pmax = 0;
    int64_t pmax_rf[KA_MAX_SLOTS + 1] = {};   // [rf] partitions of the largest topic with target RF rf (rf <= S)
    std::vector<std::pair<int, int64_t>> over;   // (t, target RF) of topics with target RF > S, each below every earlier one
    ka_status err{KA_OK, -1, -1, 0, 0};
};

// row0 / rep0: the scan reads part_off[t] - row0 and rep_off[g] - rep0, i.e. a slice of a larger layout rebased to 0 (one
// cluster of ka_solve_clusters' fleet), without copying it.
static int ragged_scan(int32_t T, const int64_t* part_off, const int64_t* rep_off, const int32_t* cur_broker, int32_t desired_rf,
                       int32_t S, int pick_max, bool have_out, RaggedScan& sc, ka_status* st, int64_t row0 = 0, int64_t rep0 = 0) {
    const int64_t Q = T > 0 ? part_off[T] - row0 : 0;
    if (Q < 0 || (T > 0 && part_off[0] != row0) || (Q > 0 && (!rep_off || !have_out))) return set_status(st, KA_ERR_BAD_ARG);
    const int64_t R = Q > 0 ? rep_off[Q] - rep0 : 0;
    if (R < 0 || (Q > 0 && rep_off[0] != rep0) || (R > 0 && !cur_broker)) return set_status(st, KA_ERR_BAD_ARG);
    if (pick_max > 0) {
        int64_t m = std::max(desired_rf, 1);
        for (int64_t g = 0; g < Q; ++g) m = std::max(m, rep_off[g + 1] - rep_off[g]);
        if (m > pick_max) return set_status(st, KA_ERR_LIMIT, -1, -1, (int)std::min<int64_t>(m, INT_MAX));
        S = (int)m;
    }
    sc.Q = Q;
    sc.R = R;
    sc.S = S;
    for (int t = 0; t < T; ++t) {
        const int64_t a = part_off[t] - row0, b = part_off[t + 1] - row0;
        if (b < a) { set_status(&sc.err, KA_ERR_BAD_ARG, t); return KA_OK; }
        const int64_t Pn = b - a;
        if (Pn > INT_MAX / 16) { set_status(&sc.err, KA_ERR_LIMIT, t, -1, (int)std::min<int64_t>(Pn, INT_MAX)); return KA_OK; }
        sc.Pmax = std::max<int>(sc.Pmax, (int)Pn);
        int64_t rf_t = desired_rf;
        if (rf_t < 0 && Pn > 0) rf_t = rep_off[a + 1] - rep_off[a];
        if (rf_t > S) {
            if (sc.over.empty() || rf_t < sc.over.back().second) sc.over.emplace_back(t, rf_t);
        } else if (rf_t > 0) {
            sc.pmax_rf[rf_t] = std::max(sc.pmax_rf[rf_t], Pn);
        }
    }
    for (int64_t g = 0; g < Q; ++g) {
        const int64_t sz = rep_off[g + 1] - rep_off[g];
        if (sz < 0) { set_status(&sc.err, KA_ERR_BAD_ARG); return KA_OK; }
        sc.maxsz = std::max(sc.maxsz, sz);
    }
    if (sc.maxsz > S) set_status(&sc.err, KA_ERR_BAD_ARG, -1, -1, S);
    return KA_OK;
}

// The largest capacity (KAS:65-71) of a scanned ragged problem under a table of N brokers — over the topics whose target RF
// the table can serve — or the failure ka_solve reports for that table.
static int ragged_capmax(const RaggedScan& sc, int N, int64_t& capmax, ka_status* st) {
    capmax = 0;
    if (N > 0)
        for (const auto& o : sc.over)   // the first topic whose target RF is in (S, N]
            if (o.second <= N) return set_status(st, KA_ERR_BAD_ARG, o.first, -1, sc.S);
    if (sc.err.code != KA_OK) {
        if (st) *st = sc.err;
        return sc.err.code;
    }
    for (int rf = 1; rf <= std::min(sc.S, N); ++rf) capmax = std::max<int64_t>(capmax, (sc.pmax_rf[rf] * rf + N - 1) / N);
    return KA_OK;
}

// Validation and sizing of a ragged solve against the ctx's broker table, then its device input buffers: the Shape
// run_solve takes. pick_stride / have_out: as in ragged_scan.
static int prepare_ragged(ka_ctx* c, int32_t T, const int32_t* topic_hash, const int64_t* part_off, const int64_t* rep_off,
                          const int32_t* cur_broker, int32_t desired_rf, int32_t S, bool pick_stride, bool have_out, Shape& sh,
                          ka_status* st) {
    set_status(st, KA_OK);
    if (!c) return set_status(st, KA_ERR_NO_DEVICE);
    if (T < 0 || (T > 0 && (!topic_hash || !part_off))) return set_status(st, KA_ERR_BAD_ARG);
    if (!pick_stride && (S < 1 || S > KA_MAX_SLOTS)) return set_status(st, KA_ERR_LIMIT, -1, -1, S);
    int rc = enter_host(c);
    if (rc != KA_OK) return failed(st, rc);
    RaggedScan sc;
    int64_t capmax = 0;
    if ((rc = ragged_scan(T, part_off, rep_off, cur_broker, desired_rf, S, pick_stride ? KA_MAX_SLOTS : 0, have_out, sc, st)) != KA_OK ||
        (rc = ragged_capmax(sc, c->br.N, capmax, st)) != KA_OK)
        return rc;
    sh = ragged_shape(T, sc.Q, sc.R, desired_rf, sc.S, sc.Pmax, capmax);
    if ((rc = reserve_io(c, sh, true)) != KA_OK) return failed(st, rc);
    return KA_OK;
}

int32_t ka_solve(ka_ctx* c, int32_t T, const int32_t* topic_hash, const int64_t* part_off,
                 const int32_t* part_id, const int64_t* rep_off, const int32_t* cur_broker,
                 int32_t desired_rf, int32_t out_stride, int32_t* out_len, int32_t* out_broker,
                 ka_status* st) {
    Shape sh;
    int rc = prepare_ragged(c, T, topic_hash, part_off, rep_off, cur_broker, desired_rf, out_stride, false, out_broker != nullptr, sh, st);
    if (rc != KA_OK) return rc;
    SolveCall io = host_call(c, topic_hash, part_off, rep_off, cur_broker, out_len, out_broker);
    if ((rc = run_solve(c, c->stream, sh, io, st)) != KA_OK) return failed(st, rc);
    return finish(c, c->stream, st, true, part_id, part_off);
}

// The longest of the names of topics [t0, t1).
static int64_t longest_name(const int64_t* name_off, int t0, int t1) {
    int64_t m = 0;
    for (int t = t0; t < t1; ++t) m = std::max(m, name_off[t + 1] - name_off[t]);
    return m;
}

// A fragment's offsets are 32-bit: the rows of a fragment of a Q-row text at their longest (any int32 partition id, S
// replicas, the longest name) must fit, else KA_ERR_LIMIT with a = the longest name.
static int check_fragments(int64_t Q, int S, int64_t longest, ka_status* st) {
    const int64_t frag_rows = std::min(json_fragment_rows(Q), std::max<int64_t>(Q, 1));
    if (64 + frag_rows * (50 + 12 * S + longest) > (int64_t)UINT32_MAX)
        return set_status(st, KA_ERR_LIMIT, -1, -1, (int)std::min<int64_t>(longest, INT_MAX));
    return KA_OK;
}

int32_t ka_solve_json(ka_ctx* c, int32_t T, const int32_t* topic_hash, const int64_t* part_off, const int32_t* part_id,
                      const int64_t* rep_off, const int32_t* cur_broker, int32_t desired_rf, const char* names,
                      const int64_t* name_off, char* json, int64_t json_cap, int64_t* json_bytes, ka_status* st) {
    if (json_bytes) *json_bytes = 0;
    Shape sh;
    int rc = prepare_ragged(c, T, topic_hash, part_off, rep_off, cur_broker, desired_rf, 0, true, true, sh, st);
    if (rc != KA_OK) return rc;
    if ((T > 0 && (!names || !name_off)) || !json || json_cap < 0) return set_status(st, KA_ERR_BAD_ARG);
    if ((rc = check_names(names, name_off, 0, T, st)) != KA_OK) return rc;
    if ((rc = check_fragments(sh.Q, sh.S, longest_name(name_off, 0, T), st)) != KA_OK) return rc;
    if (c->d_part_id.reserve((size_t)std::max<int64_t>(sh.Q, 1) * 4) != cudaSuccess) return failed(st, KA_ERR_CUDA);
    return solve_json(c, sh, host_call(c, topic_hash, part_off, rep_off, cur_broker, nullptr, nullptr, part_id), names, name_off, json,
                      json_cap, json_bytes, st);
}

// ka_solve_candidates and ka_score_candidates once their tables have passed check_tables, up to their plan: the sizing scan,
// the stride check, the tables and the candidates (bt), and the call's device inputs and rows (sh). bt has no member when
// there is nothing to solve (T == 0). have_out: as in ragged_scan.
static int ragged_candidates(ka_ctx* c, int32_t K, const int32_t* cand_off, const int32_t* broker_id, const int32_t* broker_rack,
                             int32_t T, const int64_t* part_off, const int64_t* rep_off, const int32_t* cur_broker,
                             int32_t desired_rf, int32_t out_stride, bool have_out, Batch& bt, Shape& sh, ka_status* st) {
    if (T == 0) return KA_OK;
    // malformed offsets: every candidate reports what ka_solve reports for its table
    RaggedScan sc;
    ka_status sst{};
    int rc = ragged_scan(T, part_off, rep_off, cur_broker, desired_rf, out_stride, 0, have_out, sc, &sst);
    if (rc != KA_OK) {
        for (int k = 0; k < K; ++k) st[k] = sst;
        return rc;
    }
    // each table's capacity bound, or the status ka_solve reports for it; a table fails only with malformed offsets or a topic
    // whose target RF exceeds the stride, which the stride check below refuses for every candidate
    std::vector<int64_t> cap(K);
    for (int k = 0; k < K; ++k) ragged_capmax(sc, cand_off[k + 1] - cand_off[k], cap[k], st + k);
    if (sc.err.code != KA_OK) return st[0].code;
    // the stride holds every current list and the desired RF: every candidate's ka_solve would accept the call's input
    if (out_stride < std::max<int64_t>(sc.maxsz, desired_rf)) return fail_members(st, K, KA_ERR_BAD_ARG);
    const int64_t Q = sc.Q;
    if ((rc = batch_tables(c, K, cand_off, broker_id, broker_rack, (int64_t)K * Q, bt, st)) != KA_OK) return rc;
    add_candidates(bt, T, Q, sc.Pmax, desired_rf, cap);
    const size_t q = (size_t)std::max<int64_t>(Q, 1);
    sh = ragged_shape(T, Q, sc.R, desired_rf, out_stride);
    if (reserve_io(c, sh, true) != KA_OK || c->d_out.reserve((size_t)K * q * out_stride * 4) != cudaSuccess ||
        c->d_out_len.reserve((size_t)K * q * 4) != cudaSuccess)
        return fail_members(st, K, KA_ERR_CUDA);
    return KA_OK;
}

// The summary of a candidate that has none: failed, or T == 0.
static ka_move_summary empty_summary() {
    ka_move_summary e{};
    e.max_broker_in_id = -1;
    return e;
}

int32_t ka_solve_candidates(ka_ctx* c, int32_t K, const int32_t* cand_off, const int32_t* broker_id, const int32_t* broker_rack,
                            int32_t T, const int32_t* topic_hash, const int64_t* part_off, const int32_t* part_id,
                            const int64_t* rep_off, const int32_t* cur_broker, int32_t desired_rf, int32_t out_stride,
                            int32_t* out_len, int32_t* out_broker, ka_status* st) {
    int rc = batch_args(c, K, out_stride, st);
    if (rc != KA_OK) return rc;
    if (T < 0 || (T > 0 && (!topic_hash || !part_off))) return fail_members(st, K, KA_ERR_BAD_ARG);
    if (K == 0) return KA_OK;
    if ((rc = check_tables(K, cand_off, broker_id, broker_rack)) != KA_OK) return fail_members(st, K, rc);
    Batch bt;
    Shape sh;
    StageDesc d;
    // the inputs go up once and are shared by every candidate; the rows of all candidates come back in one copy
    if ((rc = ragged_candidates(c, K, cand_off, broker_id, broker_rack, T, part_off, rep_off, cur_broker, desired_rf, out_stride,
                                out_broker != nullptr, bt, sh, st)) != KA_OK || bt.m.empty() ||
        (rc = plan_batch(sh, bt, d, st)) != KA_OK ||
        (rc = run_batch(c, c->stream, bt, d, sh.R, host_call(c, topic_hash, part_off, rep_off, cur_broker, out_len, out_broker), st)) !=
            KA_OK)
        return rc;
    return finish_batch(c, c->stream, bt, st, part_id, part_off);
}

// A fleet call past its front end: cluster k's first row and first current replica in the shared input (row0[K] = ΣP, rep0[K]
// = ΣR), and the batch of the clusters that passed.
struct Fleet {
    int T = 0;
    std::vector<int64_t> row0, rep0;
    Batch bt;
};

// The front end of ka_solve_clusters and ka_solve_clusters_json, once batch_args has passed and K > 0: the checks of the whole
// call (tables, cluster boundaries, ΣP < 2^31), which fail every cluster; then every cluster's slice checked and sized as the
// single solve checks and sizes it against the cluster's table, and its own plan. A cluster that fails there reports what the
// single solve reports and is left out of the call. out_stride > 0: the single solve is ka_solve with that stride. out_stride
// == 0: it is ka_solve_json (names / name_off: the call's name slab); every cluster picks its width, max(longest list,
// desired RF, 1), which the batched chains take up to 3 (above: KA_ERR_LIMIT, a = the width), then its names are checked
// and its text's fragment size.
static int fleet_front(ka_ctx* c, int32_t K, const int32_t* cand_off, const int32_t* broker_id, const int32_t* broker_rack,
                       const int32_t* topic_off, const int32_t* desired_rf, const int32_t* topic_hash, const int64_t* part_off,
                       const int64_t* rep_off, const int32_t* cur_broker, int32_t out_stride, bool have_out, const char* names,
                       const int64_t* name_off, Fleet& f, ka_status* st) {
    int rc;
    if ((rc = check_tables(K, cand_off, broker_id, broker_rack)) != KA_OK) return fail_members(st, K, rc);
    // the clusters' boundaries: topic_off, then part_off at their first topics and rep_off at their first rows, each
    // non-decreasing from 0
    if (!topic_off || topic_off[0] != 0) return fail_members(st, K, KA_ERR_BAD_ARG);
    for (int k = 0; k < K; ++k)
        if (topic_off[k + 1] < topic_off[k]) return fail_members(st, K, KA_ERR_BAD_ARG);
    const int T = f.T = topic_off[K];
    if (T > 0 && (!topic_hash || !part_off)) return fail_members(st, K, KA_ERR_BAD_ARG);
    std::vector<int64_t>& row0 = f.row0;
    std::vector<int64_t>& rep0 = f.rep0;
    row0.assign(K + 1, 0);
    rep0.assign(K + 1, 0);
    for (int k = 0; k <= K; ++k) {
        row0[k] = T > 0 ? part_off[topic_off[k]] : 0;
        if (row0[k] < (k > 0 ? row0[k - 1] : 0) || row0[0] != 0) return fail_members(st, K, KA_ERR_BAD_ARG);
    }
    const int64_t Q = row0[K];
    if (Q > 0 && !rep_off) return fail_members(st, K, KA_ERR_BAD_ARG);
    for (int k = 0; k <= K; ++k) {
        rep0[k] = Q > 0 ? rep_off[row0[k]] : 0;
        if (rep0[k] < (k > 0 ? rep0[k - 1] : 0) || rep0[0] != 0) return fail_members(st, K, KA_ERR_BAD_ARG);
    }
    if (Q >= ((int64_t)1 << 31)) return fail_members(st, K, KA_ERR_LIMIT);
    const bool json = out_stride == 0;
    if (json && T > 0 && (!names || !name_off)) return fail_members(st, K, KA_ERR_BAD_ARG);
    std::vector<BatchMember> passed;
    for (int k = 0; k < K; ++k) {
        const int t0 = topic_off[k];
        BatchMember mb{k, t0, topic_off[k + 1] - t0, row0[k], 0, desired_rf ? desired_rf[k] : -1, row0[k], t0};
        mb.n = cand_off[k + 1] - cand_off[k];
        RaggedScan sc;
        if (ragged_scan(mb.T, part_off ? part_off + t0 : nullptr, rep_off ? rep_off + row0[k] : nullptr,
                        cur_broker ? cur_broker + rep0[k] : nullptr, mb.desired_rf, out_stride, json ? 3 : 0, have_out, sc,
                        st + k, row0[k], rep0[k]) != KA_OK ||
            ragged_capmax(sc, mb.n, mb.capmax, st + k) != KA_OK)
            continue;
        if (json && (check_names(names, name_off, t0, t0 + mb.T, st + k) != KA_OK ||
                     check_fragments(sc.Q, sc.S, longest_name(name_off, t0, t0 + mb.T), st + k) != KA_OK))
            continue;
        mb.Q = sc.Q;
        mb.Pmax = sc.Pmax;
        mb.S = sc.S;
        passed.push_back(mb);
    }
    if ((rc = batch_tables(c, K, cand_off, broker_id, broker_rack, Q, f.bt, st)) != KA_OK) return rc;
    add_clusters(f.bt, T, Q, passed, st);
    return KA_OK;
}

int32_t ka_solve_clusters(ka_ctx* c, int32_t K, const int32_t* cand_off, const int32_t* broker_id, const int32_t* broker_rack,
                          const int32_t* topic_off, const int32_t* desired_rf, const int32_t* topic_hash, const int64_t* part_off,
                          const int32_t* part_id, const int64_t* rep_off, const int32_t* cur_broker, int32_t out_stride,
                          int32_t* out_len, int32_t* out_broker, ka_status* st) {
    int rc = batch_args(c, K, out_stride, st);
    if (rc != KA_OK) return rc;
    if (K == 0) return KA_OK;
    Fleet f;
    if ((rc = fleet_front(c, K, cand_off, broker_id, broker_rack, topic_off, desired_rf, topic_hash, part_off, rep_off, cur_broker,
                          out_stride, out_broker != nullptr, nullptr, nullptr, f, st)) != KA_OK)
        return rc;
    Batch& bt = f.bt;
    if (bt.m.empty()) return finish_batch(c, c->stream, bt, st);
    Shape sh = ragged_shape(f.T, f.row0[K], f.rep0[K], -1, out_stride);
    if (reserve_io(c, sh, true) != KA_OK) return fail_members(st, K, KA_ERR_CUDA);
    // the inputs of every cluster go up at once; the rows of all clusters come back in one copy
    StageDesc d;
    if ((rc = plan_batch(sh, bt, d, st)) != KA_OK ||
        (rc = run_batch(c, c->stream, bt, d, sh.R, host_call(c, topic_hash, part_off, rep_off, cur_broker, out_len, out_broker), st)) !=
            KA_OK)
        return rc;
    return finish_batch(c, c->stream, bt, st, part_id, part_off);
}

// The document table of a fleet's segmented JSON pass in d_json_seg: the arrays of KaJsonSegs.
struct FleetSegs { unsigned long long *doc_off, *bytes; int64_t* row0; uint32_t* shift; int32_t* member; };
static auto fleet_segs_layout(int K) {
    return [K](Layout& l) {
        return FleetSegs{l.take<unsigned long long>(K + 1), l.take<unsigned long long>(K), l.take<int64_t>(K + 1), l.take<uint32_t>(K),
                         l.take<int32_t>(K)};
    };
}

// The K clusters' first rows and batch members (-1: left out) to the document table, bytes zeroed, on `s`.
static int enq_fleet_segs(ka_ctx* c, cudaStream_t s, const Fleet& f, int K) {
    std::vector<unsigned char> h(layout_bytes(fleet_segs_layout(K)), 0);
    const FleetSegs hs = place(fleet_segs_layout(K), h.data());
    std::copy(f.row0.begin(), f.row0.begin() + K + 1, hs.row0);
    std::fill(hs.member, hs.member + K, -1);
    for (size_t i = 0; i < f.bt.m.size(); ++i) hs.member[f.bt.m[i].tab] = (int32_t)i;
    KA_CUDA(c->d_json_seg.reserve(h.size()));
    KA_CUDA(cudaMemcpyAsync(c->d_json_seg.p, h.data(), h.size(), cudaMemcpyHostToDevice, s));
    return KA_OK;
}

// The kernels' view of the K clusters' table that enq_fleet_segs uploaded, with the batch's failure words.
static KaJsonSegs fleet_segs(ka_ctx* c, int K) {
    const FleetSegs sg = place(fleet_segs_layout(K), c->d_json_seg.p);
    return KaJsonSegs{K, sg.row0, sg.member, c->batch_run.flags.as<unsigned>(), sg.bytes, sg.doc_off, sg.shift};
}

// The segmented JSON pass of a fleet solved as d (its rows in io.d_out, its document table uploaded), on `s` after the last
// emit: the length pass and the scan over fragments of the call's rows, the document table, then the write pass. doc_off
// comes back to h_doc.
static int enq_fleet_json(ka_ctx* c, cudaStream_t s, const StageDesc& d, const SolveCall& io, int K, unsigned long long* h_doc) {
    const KaJsonSegs sg = fleet_segs(c, K);
    // fragments of whole 256-row blocks, as in a ragged single solve; their count depends on the rows alone
    const int64_t Q = d.Q, step = json_fragment_rows(Q);
    std::vector<KaJsonParams> frags;
    for (int64_t r = 0; r < Q; r += step) {
        frags.push_back(json_fragment(c, d, io, r, std::min(step, Q - r), (int)frags.size()));
        enq_json_lengths<true>(s, frags.back(), sg);
    }
    ka_json_docs_kernel<<<1, KA_JSON_MAX_SEGS, 0, s>>>(json_fragment(c, d, io, 0, Q, 0), sg);   // reads json and cap alone
    for (const KaJsonParams& fp : frags) KA_CUDA(enq_json_write(ka_json_write_kernel<true>, (fp.Q + 255) / 256, s, fp, sg));
    KA_CUDA(cudaGetLastError());
    c->launches += 3 * (int64_t)frags.size() + 1;
    KA_CUDA(cudaMemcpyAsync(h_doc, sg.doc_off, (size_t)(K + 1) * 8, cudaMemcpyDeviceToHost, s));
    return KA_OK;
}

int32_t ka_solve_clusters_json(ka_ctx* c, int32_t K, const int32_t* cand_off, const int32_t* broker_id, const int32_t* broker_rack,
                               const int32_t* topic_off, const int32_t* desired_rf, const int32_t* topic_hash, const int64_t* part_off,
                               const int32_t* part_id, const int64_t* rep_off, const int32_t* cur_broker, const char* names,
                               const int64_t* name_off, char* json, int64_t json_cap, int64_t* json_off, ka_status* st) {
    if (json_off && K >= 0) std::fill(json_off, json_off + K + 1, 0);
    int rc = batch_args(c, K, 1, st);
    if (rc != KA_OK) return rc;
    if (!json || !json_off || json_cap < 0) return fail_members(st, K, KA_ERR_BAD_ARG);
    if (K == 0) return KA_OK;
    Fleet f;
    if ((rc = fleet_front(c, K, cand_off, broker_id, broker_rack, topic_off, desired_rf, topic_hash, part_off, rep_off, cur_broker, 0,
                          true, names, name_off, f, st)) != KA_OK)
        return rc;
    Batch& bt = f.bt;
    // every cluster's document, placed as the device places them: a failed cluster's range is empty
    std::vector<unsigned long long> doc(K + 1, 0);
    if (bt.m.empty()) {   // no topic to solve: every cluster that passed gets the empty document
        for (int k = 0; k < K; ++k) doc[k + 1] = doc[k] + (st[k].code == KA_OK ? KA_JSON_HEAD_LEN + KA_JSON_TAIL_LEN : 0);
        if ((int64_t)doc[K] <= json_cap)
            for (int k = 0; k < K; ++k)
                if (doc[k + 1] > doc[k]) std::memcpy(json + doc[k], KA_JSON_HEAD KA_JSON_TAIL, KA_JSON_HEAD_LEN + KA_JSON_TAIL_LEN);
    } else {
        // one plan and one stride for the call, from its largest member; a fragment size that fails where no cluster's own does
        // fails every cluster
        int S = 1;
        int64_t longest = 0;
        for (const BatchMember& mb : bt.m) {
            S = std::max(S, mb.S);
            longest = std::max(longest, longest_name(name_off, mb.t0, mb.t0 + mb.T));
        }
        Shape sh = ragged_shape(f.T, f.row0[K], f.rep0[K], -1, S);
        if ((rc = check_fragments(sh.Q, S, longest, st)) != KA_OK) {
            for (int k = 1; k < K; ++k) st[k] = st[0];
            return rc;
        }
        if (reserve_io(c, sh, true) != KA_OK || c->d_part_id.reserve((size_t)std::max<int64_t>(sh.Q, 1) * 4) != cudaSuccess)
            return fail_members(st, K, KA_ERR_CUDA);
        StageDesc d;
        if ((rc = plan_batch(sh, bt, d, st)) != KA_OK) return rc;
        // the names go up on c->sj (prepare_json), which the call's stream waits for before its first fragment
        if ((rc = prepare_json(c, f.T, sh.Q, names, name_off, json_cap)) != KA_OK ||
            cudaEventRecord(c->ev_json_in[0], c->sj) != cudaSuccess || cudaStreamWaitEvent(c->stream, c->ev_json_in[0], 0) != cudaSuccess) {
            cudaStreamSynchronize(c->sj);
            return fail_members(st, K, KA_ERR_CUDA);
        }
        if (enq_fleet_segs(c, c->stream, f, K) != KA_OK) return abort_batch(c, c->stream, st, K, KA_ERR_CUDA);
        const SolveCall io = host_call(c, topic_hash, part_off, rep_off, cur_broker, nullptr, nullptr, part_id);
        if ((rc = run_batch(c, c->stream, bt, d, sh.R, io, st)) != KA_OK) return rc;
        if ((rc = enq_fleet_json(c, c->stream, d, io, K, doc.data())) != KA_OK ||
            cudaStreamSynchronize(c->stream) != cudaSuccess ||
            ((int64_t)doc[K] <= json_cap && doc[K] > 0 && cudaMemcpy(json, c->d_json.p, doc[K], cudaMemcpyDeviceToHost) != cudaSuccess))
            return abort_batch(c, c->stream, st, K, rc != KA_OK ? rc : KA_ERR_CUDA);
        finish_batch(c, c->stream, bt, st, part_id, part_off);
    }
    // a text beyond json_cap: every cluster that solved reports the buffer, and no cluster has text
    const bool fits = (int64_t)doc[K] <= json_cap;
    for (int k = 0; k < K; ++k) {
        if (!fits && st[k].code == KA_OK) set_status(st + k, KA_ERR_LIMIT, -1, -1, (int)std::min<int64_t>(json_cap, INT_MAX));
        json_off[k + 1] = fits ? (int64_t)doc[k + 1] : 0;
    }
    for (int k = 0; k < K; ++k)
        if (st[k].code != KA_OK) return st[k].code;
    return KA_OK;
}

// What a scored call hands back when it has no result (it failed, or it has nothing to solve): every summary empty and,
// once the K tables have passed check_tables (nb = their brokers), every per-broker sum 0. Returns code.
static int score_empty(int K, ka_move_summary* summary, int64_t* const brk[3], size_t nb, int code) {
    for (int k = 0; k < K; ++k) summary[k] = empty_summary();
    for (int i = 0; i < 3; ++i)
        if (brk[i] && nb > 0) std::memset(brk[i], 0, nb * 8);
    return code;
}

// The weights of Q rows (null: none), each row adding at most `factor` x its weight to a device sum: KA_ERR_BAD_ARG when a
// weight is negative, else KA_ERR_LIMIT when factor x their sum is beyond INT64_MAX, else KA_OK. A scored call checks them
// (factor 3) once every check of its solve has passed and before anything is enqueued, ka_plan_waves (factor 8) last of its
// argument checks.
static int weights_code(const int64_t* part_weight, int64_t Q, int64_t factor) {
    if (!part_weight) return KA_OK;
    bool negative = false;
    int64_t sum = 0;   // saturates above INT64_MAX / factor
    for (int64_t g = 0; g < Q; ++g) {
        const int64_t w = part_weight[g];
        negative |= w < 0;
        sum = w > INT64_MAX / factor - sum ? INT64_MAX : sum + std::max<int64_t>(w, 0);
    }
    if (negative) return KA_ERR_BAD_ARG;
    return sum > INT64_MAX / factor ? KA_ERR_LIMIT : KA_OK;
}

// The tail of ka_score_candidates and ka_score_clusters, once run_batch has enqueued the batch bt on `s` (its rows, Q per
// candidate or ΣP for a fleet, of stride S in io.d_out): the weights and cand_off up, the accumulators zeroed, the two score
// kernels (with a fleet f, their FLEET instances over f's cluster table), the summaries and the per-broker sums asked for
// (brk) back, then finish_batch.
static int score_batch(ka_ctx* c, cudaStream_t s, const Batch& bt, const int32_t* cand_off, int64_t Q, int S, const SolveCall& io,
                       const int64_t* part_weight, const Fleet* f, ka_move_summary* summary, int64_t* const brk[3], ka_status* st,
                       const int32_t* part_id, const int64_t* part_off) {
    const int K = bt.K;
    const size_t nb = (size_t)cand_off[K];
    auto abort = [&](int code) { return score_empty(K, summary, brk, nb, abort_batch(c, s, st, K, code)); };
    const size_t sum_bytes = (size_t)K * sizeof(ka_move_summary), brk_n = std::max<size_t>(3 * nb, 1);
    // the K summaries, the per-broker sums [3][ΣN] and the tables' offsets [K+1]
    struct Scores { ka_move_summary* sum; long long* brk; int32_t* off; };
    const auto sc = reserve_layout(c->d_score, [&](Layout& l) {
        return Scores{l.take<ka_move_summary>(K), l.take<long long>(brk_n), l.take<int32_t>(K + 1)};
    });
    if (!sc || (part_weight && c->d_score_w.reserve((size_t)std::max<int64_t>(Q, 1) * 8) != cudaSuccess)) return abort(KA_ERR_CUDA);
    const auto [d_sum, d_brk, d_off] = *sc;
    const int64_t* d_w = part_weight ? c->d_score_w.as<int64_t>() : nullptr;
    if ((part_weight && Q > 0 && cudaMemcpyAsync(c->d_score_w.p, part_weight, (size_t)Q * 8, cudaMemcpyHostToDevice, s) != cudaSuccess) ||
        cudaMemcpyAsync(d_off, cand_off, (size_t)(K + 1) * 4, cudaMemcpyHostToDevice, s) != cudaSuccess ||
        cudaMemsetAsync(d_sum, 0, sum_bytes, s) != cudaSuccess || cudaMemsetAsync(d_brk, 0, brk_n * 8, s) != cudaSuccess ||
        (f && enq_fleet_segs(c, s, *f, K) != KA_OK))
        return abort(KA_ERR_CUDA);
    const KaCandidate* cand = c->d_batch_tab.as<KaCandidate>();
    const unsigned row_blocks = (unsigned)std::max<int64_t>((Q + 255) / 256, 1);
    if (f) {   // a fleet's rows are disjoint: one thread per input row, its cluster found in the table
        const KaJsonSegs sg = fleet_segs(c, K);
        ka_score_rows_kernel<true><<<row_blocks, 256, 0, s>>>(cand, d_off, (uint32_t)Q, S, io.d_out, io.d_out_len, c->d_rep_off.as<int64_t>(),
                                                              c->d_cur.as<int32_t>(), d_w, d_sum, d_brk, d_brk + nb, d_brk + 2 * nb, sg);
        ka_score_finish_kernel<true><<<K, 256, 0, s>>>(cand, d_off, d_sum, d_brk, d_brk + nb, d_brk + 2 * nb, sg);
    } else {
        ka_score_rows_kernel<false><<<dim3(row_blocks, K), 256, 0, s>>>(cand, d_off, (uint32_t)Q, S, io.d_out, io.d_out_len,
                                                                        c->d_rep_off.as<int64_t>(), c->d_cur.as<int32_t>(), d_w, d_sum,
                                                                        d_brk, d_brk + nb, d_brk + 2 * nb, KaJsonSegs{});
        ka_score_finish_kernel<false><<<K, 256, 0, s>>>(cand, d_off, d_sum, d_brk, d_brk + nb, d_brk + 2 * nb, KaJsonSegs{});
    }
    c->launches += 2;
    if (cudaGetLastError() != cudaSuccess || cudaMemcpyAsync(summary, d_sum, sum_bytes, cudaMemcpyDeviceToHost, s) != cudaSuccess)
        return abort(KA_ERR_CUDA);
    for (int i = 0; i < 3; ++i)
        if (brk[i] && nb > 0 && cudaMemcpyAsync(brk[i], d_brk + i * nb, nb * 8, cudaMemcpyDeviceToHost, s) != cudaSuccess)
            return abort(KA_ERR_CUDA);
    return finish_batch(c, s, bt, st, part_id, part_off);
}

int32_t ka_score_candidates(ka_ctx* c, int32_t K, const int32_t* cand_off, const int32_t* broker_id, const int32_t* broker_rack,
                            int32_t T, const int32_t* topic_hash, const int64_t* part_off, const int32_t* part_id,
                            const int64_t* rep_off, const int32_t* cur_broker, int32_t desired_rf, int32_t out_stride,
                            const int64_t* part_weight, ka_move_summary* summary, int64_t* broker_replicas,
                            int64_t* broker_leaders, int64_t* broker_in, int32_t* out_len, int32_t* out_broker, ka_status* st) {
    if (!st || K < 0) return KA_ERR_BAD_ARG;
    if (!summary) return fail_members(st, K, KA_ERR_BAD_ARG);
    for (int k = 0; k < K; ++k) summary[k] = empty_summary();
    int rc = batch_args(c, K, out_stride, st);
    if (rc != KA_OK) return rc;
    if (T < 0 || (T > 0 && (!topic_hash || !part_off))) return fail_members(st, K, KA_ERR_BAD_ARG);
    if (K == 0) return KA_OK;
    if ((rc = check_tables(K, cand_off, broker_id, broker_rack)) != KA_OK) return fail_members(st, K, rc);
    int64_t* const brk[3] = {broker_replicas, broker_leaders, broker_in};
    const size_t nb = (size_t)cand_off[K];
    Batch bt;
    Shape sh;
    StageDesc d;
    if ((rc = ragged_candidates(c, K, cand_off, broker_id, broker_rack, T, part_off, rep_off, cur_broker, desired_rf, out_stride, true,
                                bt, sh, st)) != KA_OK || bt.m.empty() || (rc = plan_batch(sh, bt, d, st)) != KA_OK)
        return score_empty(K, summary, brk, nb, rc);
    if ((rc = weights_code(part_weight, sh.Q, 3)) != KA_OK) return score_empty(K, summary, brk, nb, fail_members(st, K, rc));
    const SolveCall io = host_call(c, topic_hash, part_off, rep_off, cur_broker, out_len, out_broker);
    if ((rc = run_batch(c, c->stream, bt, d, sh.R, io, st)) != KA_OK) return score_empty(K, summary, brk, nb, rc);
    return score_batch(c, c->stream, bt, cand_off, sh.Q, out_stride, io, part_weight, nullptr, summary, brk, st, part_id, part_off);
}

int32_t ka_score_clusters(ka_ctx* c, int32_t K, const int32_t* cand_off, const int32_t* broker_id, const int32_t* broker_rack,
                          const int32_t* topic_off, const int32_t* desired_rf, const int32_t* topic_hash, const int64_t* part_off,
                          const int32_t* part_id, const int64_t* rep_off, const int32_t* cur_broker, int32_t out_stride,
                          const int64_t* part_weight, ka_move_summary* summary, int64_t* broker_replicas, int64_t* broker_leaders,
                          int64_t* broker_in, int32_t* out_len, int32_t* out_broker, ka_status* st) {
    if (!st || K < 0) return KA_ERR_BAD_ARG;
    if (!summary) return fail_members(st, K, KA_ERR_BAD_ARG);
    for (int k = 0; k < K; ++k) summary[k] = empty_summary();
    int rc = batch_args(c, K, out_stride, st);
    if (rc != KA_OK) return rc;
    if (K == 0) return KA_OK;
    int64_t* const brk[3] = {broker_replicas, broker_leaders, broker_in};
    Fleet f;
    if ((rc = fleet_front(c, K, cand_off, broker_id, broker_rack, topic_off, desired_rf, topic_hash, part_off, rep_off, cur_broker,
                          out_stride, true, nullptr, nullptr, f, st)) != KA_OK)
        return check_tables(K, cand_off, broker_id, broker_rack) == KA_OK ? score_empty(K, summary, brk, (size_t)cand_off[K], rc) : rc;
    const size_t nb = (size_t)cand_off[K];
    Batch& bt = f.bt;
    if (bt.m.empty()) return score_empty(K, summary, brk, nb, finish_batch(c, c->stream, bt, st));
    Shape sh = ragged_shape(f.T, f.row0[K], f.rep0[K], -1, out_stride);
    if (reserve_io(c, sh, true) != KA_OK) return score_empty(K, summary, brk, nb, fail_members(st, K, KA_ERR_CUDA));
    // the inputs of every cluster go up at once; the weights are checked over all ΣP rows
    StageDesc d;
    if ((rc = plan_batch(sh, bt, d, st)) != KA_OK) return score_empty(K, summary, brk, nb, rc);
    if ((rc = weights_code(part_weight, sh.Q, 3)) != KA_OK) return score_empty(K, summary, brk, nb, fail_members(st, K, rc));
    const SolveCall io = host_call(c, topic_hash, part_off, rep_off, cur_broker, out_len, out_broker);
    if ((rc = run_batch(c, c->stream, bt, d, sh.R, io, st)) != KA_OK) return score_empty(K, summary, brk, nb, rc);
    return score_batch(c, c->stream, bt, cand_off, sh.Q, out_stride, io, part_weight, &f, summary, brk, st, part_id, part_off);
}

// The sender part of a wave plan (ka_plan_waves_send and its JSON form): the send table id[n], the budget C and the caller's
// sender summaries, one per ka_wave_summary.
struct WaveSend {
    int32_t n;
    const int32_t* id;
    int64_t C;
    ka_wave_send_summary* summary;
};

// The row checks of a wave-row call (ka_plan_waves* and ka_wave_broker_usage) that follow its own first argument check, in this
// order: rep_off never decreases, cur_broker is there for R = rep_off[Q] > 0 brokers, stride <= KA_MAX_SLOTS, Q < 2^31.
static int wave_rows_args(int64_t Q, const int64_t* rep_off, const int32_t* cur_broker, int32_t stride, int64_t& R, ka_status* st) {
    for (int64_t g = 0; g < Q; ++g)
        if (rep_off[g + 1] < rep_off[g]) return set_status(st, KA_ERR_BAD_ARG);
    R = Q > 0 ? rep_off[Q] : 0;
    if (R > 0 && !cur_broker) return set_status(st, KA_ERR_BAD_ARG);
    if (stride > KA_MAX_SLOTS) return set_status(st, KA_ERR_LIMIT, -1, -1, stride);
    if (Q >= (int64_t)1 << 31) return set_status(st, KA_ERR_LIMIT, -1, -1, INT_MAX);
    return KA_OK;
}

// Every row's new_len[g] in 0 .. stride and, with wave, wave[g] >= 0; the lowest row g that fails is refused (st.a = g).
// W = the largest wave (0 without wave).
static int wave_lens_args(int64_t Q, int32_t stride, const int32_t* new_len, const int32_t* wave, int& W, ka_status* st) {
    W = 0;
    for (int64_t g = 0; g < Q; ++g) {
        if (new_len[g] < 0 || new_len[g] > stride || (wave && wave[g] < 0)) return set_status(st, KA_ERR_BAD_ARG, -1, -1, (int)g);
        if (wave) W = std::max(W, (int)wave[g]);
    }
    return KA_OK;
}

// The broker id the device refused in row g, if any: at the first failing position of its new list, a broker named twice or,
// with `receivers`, a receiver (a broker the current list lacks) that the ascending table id[n] lacks.
static std::optional<int32_t> refused_id(const int32_t* id, size_t n, const int64_t* rep_off, const int32_t* cur, int32_t stride,
                                         const int32_t* new_len, const int32_t* new_broker, int64_t g, bool receivers) {
    const int32_t* nb = new_broker + g * stride;
    const int32_t* cb = cur + rep_off[g];
    const int64_t m = rep_off[g + 1] - rep_off[g];
    for (int j = 0; j < new_len[g]; ++j) {
        if (std::find(nb, nb + j, nb[j]) != nb + j) return nb[j];
        if (receivers && std::find(cb, cb + m, nb[j]) == cb + m && !std::binary_search(id, id + n, nb[j])) return nb[j];
    }
    return std::nullopt;
}

// The argument checks of ka_plan_waves, in its order, once st and the ctx are there. R = the current lists' brokers, positions
// = the new lists' (a bound on the chain's buckets).
static int wave_args(int64_t Q, const int64_t* rep_off, const int32_t* cur_broker, int32_t stride, const int32_t* new_len,
                     const int32_t* new_broker, const int64_t* part_weight, int64_t max_broker_in, const int32_t* n_waves,
                     const ka_wave_summary* summary, int32_t summary_cap, int64_t& R, int64_t& positions, ka_status* st) {
    if (Q < 0 || stride < 1 || !n_waves || summary_cap < 0 || (!summary && summary_cap > 0) || max_broker_in < 1 ||
        (Q > 0 && (!rep_off || !new_len || !new_broker)) || (rep_off && rep_off[0] != 0))
        return set_status(st, KA_ERR_BAD_ARG);
    int rc, W;   // the rows have no waves yet: W stays 0
    if ((rc = wave_rows_args(Q, rep_off, cur_broker, stride, R, st)) != KA_OK ||
        (rc = wave_lens_args(Q, stride, new_len, nullptr, W, st)) != KA_OK)
        return rc;
    positions = 0;
    for (int64_t g = 0; g < Q; ++g) positions += new_len[g];
    rc = weights_code(part_weight, Q, 8);   // a row adds at most 8 x its weight to a wave
    return rc != KA_OK ? set_status(st, rc) : KA_OK;
}

// The checks a sender part adds, in this order, after every check of the call without one. The 16-bit sender index of a record
// holds 0 .. 65534; 65535 marks a row without a sender.
static int wave_send_args(const WaveSend& sd, int32_t summary_cap, ka_status* st) {
    if (sd.C < 1 || sd.n < 0 || (!sd.id && sd.n > 0) || (!sd.summary && summary_cap > 0)) return set_status(st, KA_ERR_BAD_ARG);
    for (int32_t i = 1; i < sd.n; ++i)
        if (sd.id[i] <= sd.id[i - 1]) return set_status(st, KA_ERR_BAD_ARG);
    if (sd.n > (int32_t)KA_WAVE_NO_SENDER) return set_status(st, KA_ERR_LIMIT, -1, -1, sd.n);
    return KA_OK;
}

// The Q > 0 rows of a wave-row call (ka_plan_waves*, ka_wave_broker_usage) up on c->stream, into d_rep_off, d_cur (R brokers),
// d_out_len, d_out, d_score_w (weights, null: none) and d_wv_wave (waves, null: none). These buffers belong to the synchronous
// host-buffer calls (solves, scores, wave plans, broker usage): one call may overwrite what another left there, because each
// awaits its own work before it returns.
static int upload_wave_rows(ka_ctx* c, int64_t Q, int64_t R, const int64_t* rep_off, const int32_t* cur_broker, int32_t stride,
                            const int32_t* new_len, const int32_t* new_broker, const int64_t* part_weight, const int32_t* wave) {
    cudaStream_t s = c->stream;
    const size_t q = (size_t)Q;
    if (c->d_rep_off.reserve((q + 1) * 8) || c->d_cur.reserve((size_t)std::max<int64_t>(R, 1) * 4) || c->d_out_len.reserve(q * 4) ||
        c->d_out.reserve(q * stride * 4) || (part_weight && c->d_score_w.reserve(q * 8)) || (wave && c->d_wv_wave.reserve(q * 4)) ||
        cudaMemcpyAsync(c->d_rep_off.p, rep_off, (q + 1) * 8, cudaMemcpyHostToDevice, s) ||
        (R > 0 && cudaMemcpyAsync(c->d_cur.p, cur_broker, (size_t)R * 4, cudaMemcpyHostToDevice, s)) ||
        cudaMemcpyAsync(c->d_out_len.p, new_len, q * 4, cudaMemcpyHostToDevice, s) ||
        cudaMemcpyAsync(c->d_out.p, new_broker, q * stride * 4, cudaMemcpyHostToDevice, s) ||
        (part_weight && cudaMemcpyAsync(c->d_score_w.p, part_weight, q * 8, cudaMemcpyHostToDevice, s)) ||
        (wave && cudaMemcpyAsync(c->d_wv_wave.p, wave, q * 4, cudaMemcpyHostToDevice, s)))
        return KA_ERR_CUDA;
    return KA_OK;
}

// The most bytes the load table of a first-fit plan may take: Wb x (N + n_send) x 8 (kassign_waves.cuh).
constexpr size_t KA_WAVE_FIT_MAX_BYTES = size_t(1) << 30;

// The first-fit chain of wave_plan_device (KA_WAVE_FIRST_FIT), after its rows / scan / compact kernels: the counts and the
// bound Wb, awaited; unless the rows pass failed a row (left for the caller to report), KA_ERR_LIMIT with a = Wb when the load
// table exceeds KA_WAVE_FIT_MAX_BYTES, else the zeroed table, the chain (its per-row words at state, or when state is null in
// smem bytes of shared memory) and the bucket logs (the meta words' nlog / nslog).
static int wave_fit_chain(ka_ctx* c, cudaStream_t s, unsigned nblk, int N, int ns, int64_t B, bool send, unsigned char* state,
                          size_t smem, const KaWaveRec* d_rec, const int32_t* d_off, int32_t* d_wave, KaWaveBucket* d_log,
                          KaWaveMeta* d_meta, ka_status* st) {
    const size_t rows = (size_t)(N + ns);
    int* d_cnt = c->d_wv_state.as<int>();   // R_b, S_s; then, with the state in global memory, the chain's claim and hint words
    if (cudaMemsetAsync(d_cnt, 0, rows * 4, s)) return set_status(st, KA_ERR_CUDA);
    const auto count = send ? ka_wave_fit_count_kernel<true> : ka_wave_fit_count_kernel<false>;
    const auto bound = send ? ka_wave_fit_bound_kernel<true> : ka_wave_fit_bound_kernel<false>;
    count<<<nblk, 256, 0, s>>>(d_rec, d_off, (int)nblk, N, d_cnt, d_meta);
    bound<<<nblk, 256, 0, s>>>(d_rec, d_off, (int)nblk, N, d_cnt, d_meta);
    c->launches += 2;
    KaWaveMeta fm;
    if (cudaGetLastError() != cudaSuccess || cudaMemcpyAsync(&fm, d_meta, sizeof(fm), cudaMemcpyDeviceToHost, s) ||
        cudaStreamSynchronize(s))
        return set_status(st, KA_ERR_CUDA);
    if (fm.err_row != 0xFFFFFFFFu) return KA_OK;
    const int Wb = fm.bound;
    const size_t bytes = (size_t)Wb * rows * 8;
    if (bytes > KA_WAVE_FIT_MAX_BYTES) return set_status(st, KA_ERR_LIMIT, -1, -1, Wb);
    if (c->d_wv_fit.reserve(std::max<size_t>(bytes, 16)) || cudaMemsetAsync(c->d_wv_fit.p, 0, bytes, s)) return set_status(st, KA_ERR_CUDA);
    long long* table = c->d_wv_fit.as<long long>();
    const auto chain = state ? (send ? ka_wave_fit_chain_kernel<true, true> : ka_wave_fit_chain_kernel<true, false>)
                             : (send ? ka_wave_fit_chain_kernel<false, true> : ka_wave_fit_chain_kernel<false, false>);
    if (!state && allow_smem(chain, smem) != cudaSuccess) return set_status(st, KA_ERR_CUDA);
    chain<<<1, KA_WAVE_THREADS, smem, s>>>(d_rec, d_off, (int)nblk, N, (int)rows, B, Wb, d_wave, table, state, d_meta);
    const size_t n = (size_t)Wb * rows;
    const unsigned blocks = (unsigned)std::max<size_t>(1, std::min<size_t>((n + 255) / 256, (size_t)c->sm_count * 8));
    const auto log = send ? ka_wave_fit_log_kernel<true> : ka_wave_fit_log_kernel<false>;
    log<<<blocks, 256, 0, s>>>(table, Wb, N, n, d_log, d_meta);
    c->launches += 2;
    return KA_OK;
}

// The device part of a wave plan of Q > 0 checked rows, on c->stream of the entered ctx: the rows up (upload_wave_rows), the
// rows / scan / compact / chain kernels under the ctx's wave rule (KA_WAVE_FIRST_FIT: wave_fit_chain), the meta words back,
// then the sum and the two peak kernels (enqueued, not awaited).
// Leaves every row's wave in d_wv_wave, its receivers (int8, -1 unchanged) at the start of d_wv_plan, where the part caps read
// them (enq_wave_parts), the new lists in d_out / d_out_len and the W summaries (ids still N - index) in d_wv_sum. A sender part
// sd (null: none) adds the sender rule and its summaries (ids still n - index) in d_wv_ssum.
static int wave_plan_device(ka_ctx* c, int64_t Q, int64_t R, int64_t positions, const int64_t* rep_off, const int32_t* cur_broker,
                            int32_t stride, const int32_t* new_len, const int32_t* new_broker, const int64_t* part_weight,
                            int64_t max_broker_in, const WaveSend* sd, int& W, ka_status* st) {
    cudaStream_t s = c->stream;
    const int N = c->br.N;
    const int ns = sd ? sd->n : 0;
    const unsigned nblk = (unsigned)((Q + 255) / 256);
    const bool fit = c->wave_rule == KA_WAVE_FIRST_FIT;
    // the chain's per-row words (the brokers', then the senders'): in shared memory while they fit, else in d_wv_state
    const size_t state_bytes = (size_t)(N + ns) * (fit ? KA_WAVE_FIT_ROW_BYTES : KA_WAVE_ROW_BYTES);
    const bool gstate = state_bytes > KA_SMEM_BUDGET;
    const size_t q = (size_t)Q;
    // the rows pass's receiver counts and records, the packed records, the per-CTA counts, their offsets followed by their
    // total, the bucket log and the meta words
    struct PlanScratch { int8_t* nrecv; KaWaveRec *tmp, *rec; int32_t *cnt, *off; KaWaveBucket* log; KaWaveMeta* meta; };
    const auto sc = reserve_layout(c->d_wv_plan, [&](Layout& l) {
        return PlanScratch{l.take<int8_t>(q), l.take<KaWaveRec>(q), l.take<KaWaveRec>(q), l.take<int32_t>(nblk), l.take<int32_t>(nblk + 1),
                           l.take<KaWaveBucket>((size_t)std::max<int64_t>(positions, 1)), l.take<KaWaveMeta>(1)};
    });
    if (upload_wave_rows(c, Q, R, rep_off, cur_broker, stride, new_len, new_broker, part_weight, nullptr) != KA_OK || !sc ||
        c->d_wv_wave.reserve(q * 4) || c->d_wv_state.reserve(gstate || fit ? state_bytes : 16))
        return set_status(st, KA_ERR_CUDA);
    unsigned char* state = gstate ? c->d_wv_state.as<unsigned char>() : nullptr;
    const size_t smem = gstate ? 0 : state_bytes;
    // a sender bucket holds at least one moved row: at most Q of them
    if (sd && (c->d_wv_send.reserve((size_t)std::max(ns, 1) * 4) || c->d_wv_slog.reserve(q * sizeof(KaWaveBucket)) ||
               (ns > 0 && cudaMemcpyAsync(c->d_wv_send.p, sd->id, (size_t)ns * 4, cudaMemcpyHostToDevice, s))))
        return set_status(st, KA_ERR_CUDA);
    KaWaveMeta meta0{0xFFFFFFFFu, 0, 0, 0, 0, 0, {}};   // the sender part only read with sd
    if (sd) meta0.snd = KaWaveSend{c->d_wv_send.as<int32_t>(), ns, sd->C, c->d_wv_slog.as<KaWaveBucket>()};
    const int64_t* d_w = part_weight ? c->d_score_w.as<int64_t>() : nullptr;
    const auto [d_nrecv, d_tmp, d_rec, d_cnt, d_off, d_log, d_meta] = *sc;
    if (cudaMemcpyAsync(d_meta, &meta0, sizeof(meta0), cudaMemcpyHostToDevice, s)) return set_status(st, KA_ERR_CUDA);
    int32_t* d_wave = c->d_wv_wave.as<int32_t>();
    const auto rows = sd ? ka_wave_rows_kernel<true> : ka_wave_rows_kernel<false>;
    rows<<<nblk, 256, 0, s>>>(c->br, (uint32_t)Q, stride, c->d_rep_off.as<int64_t>(), c->d_cur.as<int32_t>(), c->d_out_len.as<int32_t>(),
                              c->d_out.as<int32_t>(), d_w, d_nrecv, d_tmp, d_wave, d_cnt, d_meta);
    ka_level_scan_kernel<<<1, 1024, 0, s>>>(d_cnt, (int)nblk, d_off);
    ka_wave_compact_kernel<<<nblk, 256, 0, s>>>((uint32_t)Q, d_nrecv, d_tmp, d_off, d_rec);
    c->launches += 3;   // rows, scan, compact
    if (fit) {
        int rc = wave_fit_chain(c, s, nblk, N, ns, max_broker_in, sd != nullptr, state, smem, d_rec, d_off, d_wave, d_log, d_meta, st);
        if (rc != KA_OK) return rc;
    } else {
        const auto chain = gstate ? (sd ? ka_wave_chain_kernel<true, true> : ka_wave_chain_kernel<true, false>)
                                  : (sd ? ka_wave_chain_kernel<false, true> : ka_wave_chain_kernel<false, false>);
        if (!gstate && allow_smem(chain, smem) != cudaSuccess) return set_status(st, KA_ERR_CUDA);
        chain<<<1, KA_WAVE_THREADS, smem, s>>>(d_rec, d_off, (int)nblk, N, N + ns, max_broker_in, d_wave, state, d_log, d_meta);
        c->launches += 1;
    }
    KaWaveMeta meta;
    if (cudaGetLastError() != cudaSuccess || cudaMemcpyAsync(&meta, d_meta, sizeof(meta), cudaMemcpyDeviceToHost, s) ||
        cudaStreamSynchronize(s))
        return set_status(st, KA_ERR_CUDA);
    if (meta.err_row != 0xFFFFFFFFu) {   // no refused position: with a sender part, the row's sender, which the send table lacks
        const auto id = refused_id(c->broker_id.data(), c->broker_id.size(), rep_off, cur_broker, stride, new_len, new_broker,
                                   meta.err_row, true);
        return set_status(st, KA_ERR_BAD_ARG, -1, -1, (int)meta.err_row, id ? *id : sd ? cur_broker[rep_off[meta.err_row]] : 0);
    }
    W = std::max(meta.waves, meta.changed);
    const size_t sum_bytes = (size_t)std::max(W, 1) * sizeof(ka_wave_summary);
    const size_t ssum_bytes = (size_t)std::max(W, 1) * sizeof(ka_wave_send_summary);
    if (c->d_wv_sum.reserve(sum_bytes) || (sd && c->d_wv_ssum.reserve(ssum_bytes))) return set_status(st, KA_ERR_CUDA);
    ka_wave_summary* d_sum = c->d_wv_sum.as<ka_wave_summary>();
    if (cudaMemsetAsync(d_sum, 0, sum_bytes, s) || (sd && cudaMemsetAsync(c->d_wv_ssum.p, 0, ssum_bytes, s)))
        return set_status(st, KA_ERR_CUDA);
    ka_wave_sum_kernel<<<nblk, 256, 0, s>>>((uint32_t)Q, d_nrecv, d_wave, d_w, d_sum);
    c->launches += 1;
    enq_wave_peaks<KaWaveInPeak>(c, s, d_log, meta.nlog, N, d_sum);
    if (sd) enq_wave_peaks<KaWaveOutPeak>(c, s, c->d_wv_slog.as<KaWaveBucket>(), meta.nslog, ns, c->d_wv_ssum.as<ka_wave_send_summary>());
    return cudaGetLastError() != cudaSuccess ? set_status(st, KA_ERR_CUDA) : KA_OK;
}

// The plan of wave_plan_device out to the caller: the first min(W, summary_cap) summaries (and with a sender part sd, sender
// summaries) and every row's wave, awaited; then the summaries' broker ids and *n_waves.
static int wave_plan_out(ka_ctx* c, int64_t Q, int W, int32_t* wave, int32_t* n_waves, ka_wave_summary* summary, int32_t summary_cap,
                         const WaveSend* sd, ka_status* st) {
    cudaStream_t s = c->stream;
    const int N = c->br.N;
    const int out = std::min(W, summary_cap);
    if ((out > 0 && cudaMemcpyAsync(summary, c->d_wv_sum.p, (size_t)out * sizeof(ka_wave_summary), cudaMemcpyDeviceToHost, s)) ||
        (sd && out > 0 &&
         cudaMemcpyAsync(sd->summary, c->d_wv_ssum.p, (size_t)out * sizeof(ka_wave_send_summary), cudaMemcpyDeviceToHost, s)) ||
        (wave && cudaMemcpyAsync(wave, c->d_wv_wave.p, (size_t)Q * 4, cudaMemcpyDeviceToHost, s)) || cudaStreamSynchronize(s))
        return set_status(st, KA_ERR_CUDA);
    for (int v = 0; v < out; ++v) {   // N - the lowest broker index of the wave's peak, 0 when nothing was added
        const int64_t f = summary[v].max_broker_in_id;
        summary[v].max_broker_in_id = f > 0 ? c->broker_id[N - f] : -1;
        if (sd) {   // likewise n - the lowest send-table index
            const int64_t h = sd->summary[v].max_broker_out_id;
            sd->summary[v].max_broker_out_id = h > 0 ? sd->id[sd->n - h] : -1;
        }
    }
    *n_waves = W;
    return set_status(st, KA_OK);
}

// ka_plan_waves, and with a sender part sd ka_plan_waves_send.
static int32_t plan_waves(ka_ctx* c, int64_t Q, const int64_t* rep_off, const int32_t* cur_broker, int32_t stride, const int32_t* new_len,
                          const int32_t* new_broker, const int64_t* part_weight, int64_t max_broker_in, int32_t* wave, int32_t* n_waves,
                          ka_wave_summary* summary, int32_t summary_cap, const WaveSend* sd, ka_status* st) {
    if (!st) return KA_ERR_BAD_ARG;
    if (n_waves) *n_waves = 0;
    if (!c) return set_status(st, KA_ERR_NO_DEVICE);
    int64_t R = 0, positions = 0;
    int rc = wave_args(Q, rep_off, cur_broker, stride, new_len, new_broker, part_weight, max_broker_in, n_waves, summary, summary_cap, R,
                       positions, st);
    if (rc != KA_OK) return rc;
    if (sd && (rc = wave_send_args(*sd, summary_cap, st)) != KA_OK) return rc;
    if (Q == 0) return set_status(st, KA_OK);
    // the call reads only the broker table: a pending asynchronous status stays pending for ka_last_status
    if ((rc = enter(c, false)) != KA_OK) return set_status(st, rc);
    int W = 0;
    if ((rc = wave_plan_device(c, Q, R, positions, rep_off, cur_broker, stride, new_len, new_broker, part_weight, max_broker_in, sd, W,
                               st)) != KA_OK)
        return rc;
    return wave_plan_out(c, Q, W, wave, n_waves, summary, summary_cap, sd, st);
}

int32_t ka_plan_waves(ka_ctx* c, int64_t Q, const int64_t* rep_off, const int32_t* cur_broker, int32_t stride, const int32_t* new_len,
                      const int32_t* new_broker, const int64_t* part_weight, int64_t max_broker_in, int32_t* wave, int32_t* n_waves,
                      ka_wave_summary* summary, int32_t summary_cap, ka_status* st) {
    return plan_waves(c, Q, rep_off, cur_broker, stride, new_len, new_broker, part_weight, max_broker_in, wave, n_waves, summary,
                      summary_cap, nullptr, st);
}

int32_t ka_plan_waves_send(ka_ctx* c, int64_t Q, const int64_t* rep_off, const int32_t* cur_broker, int32_t stride,
                           const int32_t* new_len, const int32_t* new_broker, const int64_t* part_weight, int64_t max_broker_in,
                           int32_t n_send, const int32_t* send_id, int64_t max_broker_out, int32_t* wave, int32_t* n_waves,
                           ka_wave_summary* summary, ka_wave_send_summary* send_summary, int32_t summary_cap, ka_status* st) {
    const WaveSend sd{n_send, send_id, max_broker_out, send_summary};
    return plan_waves(c, Q, rep_off, cur_broker, stride, new_len, new_broker, part_weight, max_broker_in, wave, n_waves, summary,
                      summary_cap, &sd, st);
}

// The tiling of a radix pass over n items: `tile` items per CTA, ntiles >= 1 CTAs. Returns the (digit, tile) cells: the pass
// counts them, then scans the counts to their offsets followed by the offsets' total.
static int radix_tiles(int64_t n, uint32_t& tile, int& ntiles) {
    tile = (uint32_t)std::max<int64_t>(KA_RADIX_MIN_TILE, ((n + KA_RADIX_MAX_TILES - 1) / KA_RADIX_MAX_TILES + 255) / 256 * 256);
    ntiles = (int)std::max<int64_t>((n + tile - 1) / tile, 1);
    return KA_RADIX_DIGITS * ntiles;
}

// The most cells of the passes over at most n items (a tile holds at least KA_RADIX_MIN_TILE of them).
static size_t radix_cells_max(int64_t n) {
    return (size_t)KA_RADIX_DIGITS * std::max<int64_t>((n + KA_RADIX_MIN_TILE - 1) / KA_RADIX_MIN_TILE, 1);
}

// The radix passes of ka_plan_waves_json over the plan's d_wv_wave, in d_wv_sort: the changed rows end ordered by (wave, row)
// in the array returned, and the (digit, tile) offsets end with M, the changed rows, at n_rows. Null when d_wv_sort fails.
static const int32_t* enq_wave_group(ka_ctx* c, cudaStream_t s, int64_t Q, int W, const int32_t*& n_rows) {
    KaWaveSort p{};
    p.wave = c->d_wv_wave.as<int32_t>();
    p.Q = (uint32_t)Q;
    const int cells = radix_tiles(Q, p.tile, p.ntiles);
    struct Sort { int32_t *perm[2], *hist, *off; };
    const auto sc = reserve_layout(c->d_wv_sort, [&](Layout& l) {
        return Sort{{l.take<int32_t>(Q), l.take<int32_t>(Q)}, l.take<int32_t>(cells), l.take<int32_t>(cells + 1)};
    });
    if (!sc) return nullptr;
    p.n_ptr = n_rows = sc->off + cells;
    int pass = 0;
    for (; pass == 0 || W >> p.shift; ++pass, p.shift += KA_RADIX_BITS) {
        p.in = pass ? sc->perm[(pass - 1) & 1] : nullptr;
        ka_wave_sort_hist_kernel<<<p.ntiles, 256, 0, s>>>(p, sc->hist);
        ka_level_scan_kernel<<<1, 1024, 0, s>>>(sc->hist, cells, sc->off);
        ka_wave_sort_scatter_kernel<<<p.ntiles, 256, 0, s>>>(p, sc->off, sc->perm[pass & 1]);
        c->launches += 3;
    }
    return sc->perm[(pass - 1) & 1];
}

// The size limit of ka_plan_waves_json_parts: L = max_doc_bytes, and the caller's doc_wave and n_docs.
struct WaveParts {
    int64_t L;
    int32_t* doc_wave;
    int32_t* n_docs;
};

// The rollback documents of ka_plan_waves_json_parts_rollback: the caller's text buffer, its size and back_off.
struct WaveBack {
    char* back;
    int64_t cap;
    int64_t* back_off;
};

extern "C++" {   // the templates of the wave text passes
// The part passes of a size limit pt over the grouped rows of d, on s: every part start flagged in pd.start, pd.part_cnt and
// pd.doc_wave placed, or KA_ERR_LIMIT for the lowest row whose one-record document exceeds pt.L. Q rows, W > 0 waves. With BACK
// the cut is the paired cut over the rollback side's bk, and a row over-long on either side is the error. With CAPS the cut
// also keeps the ctx's part caps, over the receivers the plan left first in d_wv_plan (wave_plan_device) and the weights d_w
// (null: 1 per row).
template <bool BACK, bool CAPS>
static int enq_wave_parts(ka_ctx* c, cudaStream_t s, int64_t Q, int W, const WaveParts& pt, const KaWaveDocs& d, KaWaveDocParts& pd,
                          const KaWaveBack& bk, const int64_t* d_w, ka_status* st) {
    const size_t q = (size_t)Q;
    const unsigned nblk = (unsigned)((Q + 255) / 256);
    // S [Q + 1], err and widest (one pair: set and read back in one copy), J_0 [Q], first_pos [W + 1], part_cnt [nblk],
    // doc_wave [Q], start [Q + 1]; with CAPS A [Q + 1] and its CTA sums [nblk]
    struct Parts { unsigned long long *S, *meta; int32_t *next, *first_pos, *part_cnt, *doc_wave; uint8_t* start; unsigned long long *A, *ablk; };
    const auto sc = reserve_layout(c->d_wv_part, [&](Layout& l) {
        return Parts{l.take<unsigned long long>(q + 1), l.take<unsigned long long>(2), l.take<int32_t>(q), l.take<int32_t>((size_t)W + 1),
                     l.take<int32_t>(nblk), l.take<int32_t>(q), l.take<uint8_t>(q + 1), l.take<unsigned long long>(CAPS ? q + 1 : 0),
                     l.take<unsigned long long>(CAPS ? nblk : 0)};
    });
    if (!sc) return set_status(st, KA_ERR_CUDA);
    const long long room = std::min<int64_t>(pt.L - 28, (int64_t)1 << 62);   // S[i] + room never overflows
    const KaWaveParts pp{d, room, sc->S, sc->first_pos, sc->next, sc->start, sc->meta, sc->meta + 1};
    // M < 2^31, so i + 2^32 is past every wave's end
    const KaWaveCaps cp{c->d_wv_plan.as<int8_t>(), d_w, sc->ablk, sc->A, c->part_rows > 0 ? (unsigned long long)c->part_rows : 1ull << 32,
                        c->part_in > 0 ? (unsigned long long)c->part_in : ~0ull};
    const unsigned long long meta0[2] = {~0ull, 0ull};
    if (cudaMemcpyAsync(pp.err, meta0, sizeof(meta0), cudaMemcpyHostToDevice, s)) return set_status(st, KA_ERR_CUDA);
    ka_wave_part_len_kernel<BACK, CAPS><<<nblk, 256, 0, s>>>(pp, bk, cp);
    if constexpr (BACK && CAPS)
        ka_wave_part_scan_kernel<3><<<1, 1024, 0, s>>>(d.blockoff, bk.blockoff, (int)nblk, cp.blockoff);
    else if constexpr (BACK || CAPS)
        ka_wave_part_scan_kernel<2><<<1, 1024, 0, s>>>(d.blockoff, BACK ? bk.blockoff : cp.blockoff, (int)nblk, nullptr);
    else
        ka_wave_doc_scan_kernel<false><<<1, 1024, 0, s>>>(d.blockoff, (int)nblk, pp.S, nullptr);   // S[0] is rewritten next
    ka_wave_part_prefix_kernel<BACK, CAPS><<<nblk, 256, 0, s>>>(pp, bk, cp);
    ka_wave_part_next_kernel<BACK, CAPS><<<nblk, 256, 0, s>>>(pp, bk, cp);
    c->launches += 4;
    unsigned long long back[2];
    int32_t M = 0;
    if (cudaGetLastError() != cudaSuccess || cudaMemcpyAsync(back, pp.err, sizeof(back), cudaMemcpyDeviceToHost, s) ||
        cudaMemcpyAsync(&M, d.n_rows, 4, cudaMemcpyDeviceToHost, s) || cudaStreamSynchronize(s))
        return set_status(st, KA_ERR_CUDA);
    if (back[0] != ~0ull)
        return set_status(st, KA_ERR_LIMIT, -1, -1, (int)(back[0] >> 32), (int)std::min<unsigned long long>(back[0] & 0xFFFFFFFFull, INT_MAX));
    int K = 0;   // 2^K >= the most rows, so the most parts, of a wave
    while ((1ull << K) < back[1]) ++K;
    const unsigned mblk = (unsigned)((M + 255) / 256);
    if (K > 1 && c->d_wv_jump.reserve((size_t)(K - 1) * M * 4)) return set_status(st, KA_ERR_CUDA);
    auto level = [&](int k) { return k == 0 ? pp.next : c->d_wv_jump.as<int32_t>() + (size_t)(k - 1) * M; };
    for (int k = 1; k < K; ++k) ka_wave_part_jump_kernel<<<mblk, 256, 0, s>>>(level(k - 1), level(k), (uint32_t)M);
    for (int k = K - 1; k >= 0; --k) ka_wave_part_mark_kernel<<<mblk, 256, 0, s>>>(level(k), pp.start, (uint32_t)M);
    c->launches += K > 0 ? 2 * K - 1 : 0;
    pd.start = pp.start;
    pd.part_cnt = sc->part_cnt;
    pd.doc_wave = sc->doc_wave;
    return cudaGetLastError() != cudaSuccess ? set_status(st, KA_ERR_CUDA) : KA_OK;
}

// The length / scan / write passes of one wave text: per wave, per part of pd (PARTS), or the parts' rollback text (BACK).
template <bool PARTS, bool BACK>
static cudaError_t enq_wave_text(ka_ctx* c, cudaStream_t s, unsigned nblk, const KaWaveDocs& d, unsigned long long* total,
                                 const KaWaveDocParts& pd, const KaWaveBack& kb) {
    ka_wave_doc_len_kernel<PARTS, BACK><<<nblk, 256, 0, s>>>(d, pd, kb);
    ka_wave_doc_scan_kernel<PARTS && !BACK><<<1, 1024, 0, s>>>(d.blockoff, (int)nblk, total, PARTS && !BACK ? pd.part_cnt : nullptr);
    const cudaError_t e = enq_json_write(ka_wave_doc_write_kernel<PARTS, BACK>, nblk, s, d, total, pd, kb);
    if (e == cudaSuccess) c->launches += 3;
    return e;
}
}  // extern "C++"

// ka_plan_waves_json, with a sender part sd ka_plan_waves_send_json, with a size limit pt their _parts forms, and with the
// rollback documents bk (only with pt) the _parts_rollback forms.
static int32_t plan_waves_json(ka_ctx* c, int32_t T, const int64_t* part_off, const int32_t* part_id, const int64_t* rep_off,
                               const int32_t* cur_broker, int32_t stride, const int32_t* new_len, const int32_t* new_broker,
                               const int64_t* part_weight, int64_t max_broker_in, const char* names, const int64_t* name_off, char* json,
                               int64_t json_cap, int64_t* doc_off, int32_t* wave, int32_t* n_waves, ka_wave_summary* summary,
                               int32_t summary_cap, const WaveSend* sd, const WaveParts* pt, const WaveBack* bk, ka_status* st) {
    if (!st) return KA_ERR_BAD_ARG;
    if (n_waves) *n_waves = 0;
    if (pt && pt->n_docs) *pt->n_docs = 0;
    if (!c) return set_status(st, KA_ERR_NO_DEVICE);
    if (T < 0 || (T > 0 && !part_off)) return set_status(st, KA_ERR_BAD_ARG);   // no Q to check
    const int64_t Q = T > 0 ? part_off[T] : 0;
    int64_t R = 0, positions = 0;
    int rc = wave_args(Q, rep_off, cur_broker, stride, new_len, new_broker, part_weight, max_broker_in, n_waves, summary, summary_cap, R,
                       positions, st);
    if (rc != KA_OK) return rc;
    if ((T > 0 && (part_off[0] != 0 || !names || !name_off)) || !json || json_cap < 0 || (Q > 0 && !doc_off))
        return set_status(st, KA_ERR_BAD_ARG);
    int64_t bound = 0;   // the sufficient size: per row 79 + 12 x stride + its topic's name
    int64_t back_bound = 12 * R;   // of the rollback text: per row 79 + its topic's name, 12 per current broker
    for (int t = 0; t < T; ++t) {
        if (part_off[t + 1] < part_off[t]) return set_status(st, KA_ERR_BAD_ARG);
        bound += (part_off[t + 1] - part_off[t]) * (KA_JSON_HEAD_LEN + KA_JSON_TAIL_LEN + 50 + 12 * (int64_t)stride + name_off[t + 1] - name_off[t]);
        back_bound += (part_off[t + 1] - part_off[t]) * (KA_JSON_HEAD_LEN + KA_JSON_TAIL_LEN + 50 + name_off[t + 1] - name_off[t]);
    }
    if ((rc = check_names(names, name_off, 0, T, st)) != KA_OK) return rc;
    if (sd &&(rc = wave_send_args(*sd, summary_cap, st)) != KA_OK) return rc;
    if (pt && (pt->L < 1 || (Q > 0 && (!pt->doc_wave || !pt->n_docs)))) return set_status(st, KA_ERR_BAD_ARG);
    if (bk && (!bk->back || bk->cap < 0 || (Q > 0 && !bk->back_off))) return set_status(st, KA_ERR_BAD_ARG);
    if (doc_off) doc_off[0] = 0;
    if (bk && bk->back_off) bk->back_off[0] = 0;
    if (Q == 0) return set_status(st, KA_OK);
    if ((rc = enter(c, false)) != KA_OK) return set_status(st, rc);
    int W = 0;
    if ((rc = wave_plan_device(c, Q, R, positions, rep_off, cur_broker, stride, new_len, new_broker, part_weight, max_broker_in, sd, W,
                               st)) != KA_OK)
        return rc;
    if (W == 0) return wave_plan_out(c, Q, W, wave, n_waves, summary, summary_cap, sd, st);

    cudaStream_t s = c->stream;
    const size_t q = (size_t)Q;
    const unsigned nblk = (unsigned)((Q + 255) / 256);
    const int64_t cap = std::min(json_cap, bound);
    if (c->d_part_off.reserve((size_t)(T + 1) * 8) || c->d_json.reserve((size_t)std::max<int64_t>(cap, 1)) ||
        c->d_json_rowlen.reserve(q * 4) || c->d_json_blocksum.reserve((size_t)nblk * 8) ||
        c->d_wv_doc.reserve((pt ? q + 3 : (size_t)W + 2) * 8) || upload_names(c, s, T, Q, names, name_off, part_id) != KA_OK ||
        cudaMemcpyAsync(c->d_part_off.p, part_off, (size_t)(T + 1) * 8, cudaMemcpyHostToDevice, s))
        return set_status(st, KA_ERR_CUDA);
    KaWaveDocs d{};
    d.p = json_params(c, c->d_out.as<int32_t>(), c->d_out_len.as<int32_t>(), stride, T, c->d_part_off.as<int64_t>(),
                      part_id ? c->d_part_id.as<int32_t>() : nullptr, 0, Q, (unsigned long long)cap);
    if (!(d.perm = enq_wave_group(c, s, Q, W, d.n_rows))) return set_status(st, KA_ERR_CUDA);
    d.wave = c->d_wv_wave.as<int32_t>();
    d.blockoff = c->d_json_blocksum.as<unsigned long long>();
    unsigned long long* d_total = c->d_wv_doc.as<unsigned long long>();
    d.doc_off = d_total + (pt ? 2 : 1);
    KaWaveDocParts pd{};
    // the rollback side: its row bytes [Q], CTA sums [nblk], prefix R [Q + 1], text total and back_off [Q + 1]
    struct Back { uint32_t* rowlen; unsigned long long *blockoff, *R, *total, *back_off; };
    Back bs{};
    const int64_t back_cap = bk ? std::min(bk->cap, back_bound) : 0;
    if (bk) {
        const auto sc = reserve_layout(c->d_wv_bscr, [&](Layout& l) {
            return Back{l.take<uint32_t>(q), l.take<unsigned long long>(nblk), l.take<unsigned long long>(q + 1),
                        l.take<unsigned long long>(1), l.take<unsigned long long>(q + 1)};
        });
        if (c->d_wv_back.reserve((size_t)std::max<int64_t>(back_cap, 1)) || !sc) return set_status(st, KA_ERR_CUDA);
        bs = *sc;
    }
    const KaWaveBack kb{c->d_rep_off.as<int64_t>(), c->d_cur.as<int32_t>(), bs.rowlen, bs.blockoff, bs.R};
    if (pt) {   // the caps off: the uncapped passes
        const bool caps = c->part_rows > 0 || c->part_in > 0;
        const auto parts = bk ? (caps ? enq_wave_parts<true, true> : enq_wave_parts<true, false>)
                              : (caps ? enq_wave_parts<false, true> : enq_wave_parts<false, false>);
        if ((rc = parts(c, s, Q, W, *pt, d, pd, kb, part_weight ? c->d_score_w.as<int64_t>() : nullptr, st)) != KA_OK) return rc;
    }
    const cudaError_t e = pt ? enq_wave_text<true, false>(c, s, nblk, d, d_total, pd, kb)
                             : enq_wave_text<false, false>(c, s, nblk, d, d_total, pd, kb);
    if (e != cudaSuccess) return set_status(st, KA_ERR_CUDA);
    KaWaveDocs db = d;   // the rollback text: the same positions and part starts, its own bytes, offsets, buffer and back_off
    if (bk) {
        db.p.json = c->d_wv_back.as<char>();
        db.p.cap = (unsigned long long)back_cap;
        db.p.rowlen = kb.rowlen;
        db.blockoff = kb.blockoff;
        db.doc_off = bs.back_off;
        if (enq_wave_text<true, true>(c, s, nblk, db, bs.total, pd, kb) != cudaSuccess) return set_status(st, KA_ERR_CUDA);
    }
    unsigned long long total[2] = {0, (unsigned long long)W};   // the text's bytes and the documents D
    unsigned long long back_total = 0;
    if (cudaGetLastError() != cudaSuccess || cudaMemcpyAsync(total, d_total, pt ? 16 : 8, cudaMemcpyDeviceToHost, s) ||
        (bk && cudaMemcpyAsync(&back_total, bs.total, 8, cudaMemcpyDeviceToHost, s)) || cudaStreamSynchronize(s))
        return set_status(st, KA_ERR_CUDA);
    if (total[0] > (unsigned long long)json_cap) return set_status(st, KA_ERR_LIMIT, -1, -1, (int)std::min<int64_t>(json_cap, INT_MAX));
    if (bk && back_total > (unsigned long long)bk->cap)
        return set_status(st, KA_ERR_LIMIT, -1, -1, (int)std::min<int64_t>(bk->cap, INT_MAX));
    const size_t D = (size_t)total[1];
    if (cudaMemcpyAsync(json, c->d_json.p, (size_t)total[0], cudaMemcpyDeviceToHost, s) ||
        cudaMemcpyAsync(doc_off, d.doc_off, (D + 1) * 8, cudaMemcpyDeviceToHost, s) ||
        (pt && cudaMemcpyAsync(pt->doc_wave, pd.doc_wave, D * 4, cudaMemcpyDeviceToHost, s)) ||
        (bk && (cudaMemcpyAsync(bk->back, db.p.json, (size_t)back_total, cudaMemcpyDeviceToHost, s) ||
                cudaMemcpyAsync(bk->back_off, db.doc_off, (D + 1) * 8, cudaMemcpyDeviceToHost, s))))
        return set_status(st, KA_ERR_CUDA);
    if ((rc = wave_plan_out(c, Q, W, wave, n_waves, summary, summary_cap, sd, st)) != KA_OK) return rc;
    if (pt) *pt->n_docs = (int32_t)D;
    return KA_OK;
}

int32_t ka_plan_waves_json(ka_ctx* c, int32_t T, const int64_t* part_off, const int32_t* part_id, const int64_t* rep_off,
                           const int32_t* cur_broker, int32_t stride, const int32_t* new_len, const int32_t* new_broker,
                           const int64_t* part_weight, int64_t max_broker_in, const char* names, const int64_t* name_off, char* json,
                           int64_t json_cap, int64_t* doc_off, int32_t* wave, int32_t* n_waves, ka_wave_summary* summary,
                           int32_t summary_cap, ka_status* st) {
    return plan_waves_json(c, T, part_off, part_id, rep_off, cur_broker, stride, new_len, new_broker, part_weight, max_broker_in, names,
                           name_off, json, json_cap, doc_off, wave, n_waves, summary, summary_cap, nullptr, nullptr, nullptr, st);
}

int32_t ka_plan_waves_send_json(ka_ctx* c, int32_t T, const int64_t* part_off, const int32_t* part_id, const int64_t* rep_off,
                                const int32_t* cur_broker, int32_t stride, const int32_t* new_len, const int32_t* new_broker,
                                const int64_t* part_weight, int64_t max_broker_in, int32_t n_send, const int32_t* send_id,
                                int64_t max_broker_out, const char* names, const int64_t* name_off, char* json, int64_t json_cap,
                                int64_t* doc_off, int32_t* wave, int32_t* n_waves, ka_wave_summary* summary,
                                ka_wave_send_summary* send_summary, int32_t summary_cap, ka_status* st) {
    const WaveSend sd{n_send, send_id, max_broker_out, send_summary};
    return plan_waves_json(c, T, part_off, part_id, rep_off, cur_broker, stride, new_len, new_broker, part_weight, max_broker_in, names,
                           name_off, json, json_cap, doc_off, wave, n_waves, summary, summary_cap, &sd, nullptr, nullptr, st);
}

int32_t ka_plan_waves_json_parts(ka_ctx* c, int32_t T, const int64_t* part_off, const int32_t* part_id, const int64_t* rep_off,
                                 const int32_t* cur_broker, int32_t stride, const int32_t* new_len, const int32_t* new_broker,
                                 const int64_t* part_weight, int64_t max_broker_in, const char* names, const int64_t* name_off,
                                 char* json, int64_t json_cap, int64_t max_doc_bytes, int64_t* doc_off, int32_t* doc_wave,
                                 int32_t* n_docs, int32_t* wave, int32_t* n_waves, ka_wave_summary* summary, int32_t summary_cap,
                                 ka_status* st) {
    const WaveParts pt{max_doc_bytes, doc_wave, n_docs};
    return plan_waves_json(c, T, part_off, part_id, rep_off, cur_broker, stride, new_len, new_broker, part_weight, max_broker_in, names,
                           name_off, json, json_cap, doc_off, wave, n_waves, summary, summary_cap, nullptr, &pt, nullptr, st);
}

int32_t ka_plan_waves_send_json_parts(ka_ctx* c, int32_t T, const int64_t* part_off, const int32_t* part_id, const int64_t* rep_off,
                                      const int32_t* cur_broker, int32_t stride, const int32_t* new_len, const int32_t* new_broker,
                                      const int64_t* part_weight, int64_t max_broker_in, int32_t n_send, const int32_t* send_id,
                                      int64_t max_broker_out, const char* names, const int64_t* name_off, char* json, int64_t json_cap,
                                      int64_t max_doc_bytes, int64_t* doc_off, int32_t* doc_wave, int32_t* n_docs, int32_t* wave,
                                      int32_t* n_waves, ka_wave_summary* summary, ka_wave_send_summary* send_summary,
                                      int32_t summary_cap, ka_status* st) {
    const WaveSend sd{n_send, send_id, max_broker_out, send_summary};
    const WaveParts pt{max_doc_bytes, doc_wave, n_docs};
    return plan_waves_json(c, T, part_off, part_id, rep_off, cur_broker, stride, new_len, new_broker, part_weight, max_broker_in, names,
                           name_off, json, json_cap, doc_off, wave, n_waves, summary, summary_cap, &sd, &pt, nullptr, st);
}

int32_t ka_plan_waves_json_parts_rollback(ka_ctx* c, int32_t T, const int64_t* part_off, const int32_t* part_id,
                                          const int64_t* rep_off, const int32_t* cur_broker, int32_t stride, const int32_t* new_len,
                                          const int32_t* new_broker, const int64_t* part_weight, int64_t max_broker_in,
                                          const char* names, const int64_t* name_off, char* json, int64_t json_cap,
                                          int64_t max_doc_bytes, int64_t* doc_off, int32_t* doc_wave, int32_t* n_docs, char* back,
                                          int64_t back_cap, int64_t* back_off, int32_t* wave, int32_t* n_waves,
                                          ka_wave_summary* summary, int32_t summary_cap, ka_status* st) {
    const WaveParts pt{max_doc_bytes, doc_wave, n_docs};
    const WaveBack bk{back, back_cap, back_off};
    return plan_waves_json(c, T, part_off, part_id, rep_off, cur_broker, stride, new_len, new_broker, part_weight, max_broker_in, names,
                           name_off, json, json_cap, doc_off, wave, n_waves, summary, summary_cap, nullptr, &pt, &bk, st);
}

int32_t ka_plan_waves_send_json_parts_rollback(ka_ctx* c, int32_t T, const int64_t* part_off, const int32_t* part_id,
                                               const int64_t* rep_off, const int32_t* cur_broker, int32_t stride,
                                               const int32_t* new_len, const int32_t* new_broker, const int64_t* part_weight,
                                               int64_t max_broker_in, int32_t n_send, const int32_t* send_id, int64_t max_broker_out,
                                               const char* names, const int64_t* name_off, char* json, int64_t json_cap,
                                               int64_t max_doc_bytes, int64_t* doc_off, int32_t* doc_wave, int32_t* n_docs,
                                               char* back, int64_t back_cap, int64_t* back_off, int32_t* wave, int32_t* n_waves,
                                               ka_wave_summary* summary, ka_wave_send_summary* send_summary, int32_t summary_cap,
                                               ka_status* st) {
    const WaveSend sd{n_send, send_id, max_broker_out, send_summary};
    const WaveParts pt{max_doc_bytes, doc_wave, n_docs};
    const WaveBack bk{back, back_cap, back_off};
    return plan_waves_json(c, T, part_off, part_id, rep_off, cur_broker, stride, new_len, new_broker, part_weight, max_broker_in, names,
                           name_off, json, json_cap, doc_off, wave, n_waves, summary, summary_cap, &sd, &pt, &bk, st);
}

// The argument checks of ka_wave_broker_usage, in its order, once st and the ctx are there. R = the current lists' brokers, E =
// the bound Q x stride + R on the events, W = the largest wave.
static int usage_args(int64_t Q, const int64_t* rep_off, const int32_t* cur_broker, int32_t stride, const int32_t* new_len,
                      const int32_t* new_broker, const int64_t* part_weight, const int32_t* wave, int32_t n_use, const int32_t* use_id,
                      const int64_t* use_base, const int64_t* use_cap, const ka_broker_usage* usage, const int32_t* n_waves_out,
                      int64_t& R, int64_t& E, int& W, ka_status* st) {
    if (Q < 0 || stride < 1 || n_use < 0 || (!usage && n_use > 0) || !n_waves_out ||
        (Q > 0 && (!rep_off || !new_len || !new_broker || !wave)) || (n_use > 0 && !use_id) || (rep_off && rep_off[0] != 0))
        return set_status(st, KA_ERR_BAD_ARG);
    int rc = wave_rows_args(Q, rep_off, cur_broker, stride, R, st);
    if (rc != KA_OK) return rc;
    if (n_use > 65535) return set_status(st, KA_ERR_LIMIT, -1, -1, n_use);
    for (int32_t i = 1; i < n_use; ++i)
        if (use_id[i] <= use_id[i - 1]) return set_status(st, KA_ERR_BAD_ARG);
    bool negative = false;
    for (int64_t g = 0; part_weight && g < Q; ++g) negative |= part_weight[g] < 0;
    for (int32_t i = 0; i < n_use; ++i) negative |= (use_base && use_base[i] < 0) || (use_cap && use_cap[i] < 0);
    if (negative) return set_status(st, KA_ERR_BAD_ARG);
    if ((rc = wave_lens_args(Q, stride, new_len, wave, W, st)) != KA_OK) return rc;
    // every usage is a sum of some of these terms: sum base + sum over rows of w x (current + new list lengths)
    int64_t total = 0;
    bool over = false;
    for (int32_t i = 0; use_base && i < n_use; ++i) {
        over |= use_base[i] > INT64_MAX - total;
        total = over ? INT64_MAX : total + use_base[i];
    }
    for (int64_t g = 0; g < Q && !over; ++g) {
        const int64_t w = part_weight ? part_weight[g] : 1, k = rep_off[g + 1] - rep_off[g] + new_len[g];
        over |= w > 0 && k > (INT64_MAX - total) / w;
        total = over ? INT64_MAX : total + w * k;
    }
    E = Q * stride + R;
    if (over || E > INT_MAX) return set_status(st, KA_ERR_LIMIT);
    return KA_OK;
}

int32_t ka_wave_broker_usage(ka_ctx* c, int64_t Q, const int64_t* rep_off, const int32_t* cur_broker, int32_t stride,
                             const int32_t* new_len, const int32_t* new_broker, const int64_t* part_weight, const int32_t* wave,
                             int32_t n_use, const int32_t* use_id, const int64_t* use_base, const int64_t* use_cap,
                             ka_broker_usage* usage, int32_t* n_waves_out, ka_status* st) {
    if (!st) return KA_ERR_BAD_ARG;
    if (n_waves_out) *n_waves_out = 0;
    if (!c) return set_status(st, KA_ERR_NO_DEVICE);
    int64_t R = 0, E = 0;
    int W = 0;
    int rc = usage_args(Q, rep_off, cur_broker, stride, new_len, new_broker, part_weight, wave, n_use, use_id, use_base, use_cap, usage,
                        n_waves_out, R, E, W, st);
    if (rc != KA_OK) return rc;
    // the call reads no Context state: a pending asynchronous status stays pending for ka_last_status
    if ((rc = enter(c, false)) != KA_OK) return set_status(st, rc);
    cudaStream_t s = c->stream;
    const size_t nu = (size_t)n_use;
    const unsigned nblk = (unsigned)std::max<int64_t>((Q + 255) / 256, 1);
    const size_t nu1 = std::max<size_t>(nu, 1), ne = (size_t)std::max<int64_t>(E, 1), cells_max = radix_cells_max(E);
    // the usage table's ids, bases and capacities (those given), before[], the event list twice (the radix passes' two sides),
    // the (digit, tile) counts, their offsets followed by their total, the report and the meta words
    struct Usage { int32_t* id; int64_t *base, *cap; long long* before; KaUseEvent* ev[2]; int32_t *hist, *off; ka_broker_usage* out;
                   KaUsageMeta* meta; };
    const auto u = reserve_layout(c->d_usage, [&](Layout& l) {
        return Usage{l.take<int32_t>(nu1), use_base ? l.take<int64_t>(nu + 1) : nullptr, use_cap ? l.take<int64_t>(nu + 1) : nullptr,
                     l.take<long long>(nu1), {l.take<KaUseEvent>(ne), l.take<KaUseEvent>(ne)}, l.take<int32_t>(cells_max),
                     l.take<int32_t>(cells_max + 1), l.take<ka_broker_usage>(nu1), l.take<KaUsageMeta>(1)};
    });
    if ((Q > 0 && upload_wave_rows(c, Q, R, rep_off, cur_broker, stride, new_len, new_broker, part_weight, wave) != KA_OK) || !u)
        return set_status(st, KA_ERR_CUDA);
    const KaUsageMeta meta0{0xFFFFFFFFu, 0u};
    if ((nu > 0 && cudaMemcpyAsync(u->id, use_id, nu * 4, cudaMemcpyHostToDevice, s)) ||
        (use_base && nu > 0 && cudaMemcpyAsync(u->base, use_base, nu * 8, cudaMemcpyHostToDevice, s)) ||
        (use_cap && nu > 0 && cudaMemcpyAsync(u->cap, use_cap, nu * 8, cudaMemcpyHostToDevice, s)) ||
        (nu > 0 && cudaMemsetAsync(u->before, 0, nu * 8, s)) || cudaMemcpyAsync(u->meta, &meta0, sizeof(meta0), cudaMemcpyHostToDevice, s))
        return set_status(st, KA_ERR_CUDA);
    ka_usage_rows_kernel<<<nblk, 256, 0, s>>>((uint32_t)Q, stride, c->d_rep_off.as<int64_t>(), c->d_cur.as<int32_t>(),
                                              c->d_out_len.as<int32_t>(), c->d_out.as<int32_t>(),
                                              part_weight ? c->d_score_w.as<int64_t>() : nullptr, c->d_wv_wave.as<int32_t>(), u->id, n_use,
                                              u->before, u->ev[0], u->meta);
    c->launches += 1;
    KaUsageMeta meta;
    if (cudaGetLastError() != cudaSuccess || cudaMemcpyAsync(&meta, u->meta, sizeof(meta), cudaMemcpyDeviceToHost, s) ||
        cudaStreamSynchronize(s))
        return set_status(st, KA_ERR_CUDA);
    if (meta.err_row != 0xFFFFFFFFu) {
        const auto id = refused_id(use_id, nu, rep_off, cur_broker, stride, new_len, new_broker, meta.err_row, wave[meta.err_row] > 0);
        return set_status(st, KA_ERR_BAD_ARG, -1, -1, (int)meta.err_row, id.value_or(0));
    }
    // the radix passes: the digits of the wave (1 .. W + 1), then those of the table index (0 .. n_use - 1); none without a wave
    KaUsageSort p{};
    p.ne = meta.nev;
    const int cells = radix_tiles(p.ne, p.tile, p.ntiles);
    auto bits = [](uint64_t x) { int b = 0; while (x >> b) ++b; return b; };   // x <= 2^31: the shift stays below 64
    std::vector<int> shifts;
    if (W > 0) {
        for (int b = 0; b < bits((uint64_t)W + 1); b += KA_RADIX_BITS) shifts.push_back(b);
        for (int b = 0; b < bits((uint64_t)std::max(n_use - 1, 0)); b += KA_RADIX_BITS) shifts.push_back(32 + b);
    }
    int side = 0;
    for (int shift : shifts) {
        p.in = u->ev[side];
        p.shift = shift;
        ka_usage_sort_hist_kernel<<<p.ntiles, 256, 0, s>>>(p, u->hist);
        ka_level_scan_kernel<<<1, 1024, 0, s>>>(u->hist, cells, u->off);
        ka_usage_sort_scatter_kernel<<<p.ntiles, 256, 0, s>>>(p, u->off, u->ev[side ^ 1]);
        side ^= 1;
        c->launches += 3;
    }
    ka_usage_broker_kernel<<<(unsigned)std::max<int64_t>(((int64_t)n_use + 7) / 8, 1), 256, 0, s>>>(u->ev[side], p.ne, n_use, W,
                                                                                                  u->before, u->base, u->cap, u->out);
    c->launches += 1;
    if (cudaGetLastError() != cudaSuccess ||
        (nu > 0 && cudaMemcpyAsync(usage, u->out, nu * sizeof(ka_broker_usage), cudaMemcpyDeviceToHost, s)) || cudaStreamSynchronize(s))
        return set_status(st, KA_ERR_CUDA);
    *n_waves_out = W;
    return set_status(st, KA_OK);
}

}  // extern "C"
