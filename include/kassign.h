/* kassign.h — C ABI of libkassign.so, the H100-native drop-in for ONE path of SiftScience/kafka-assigner:
 *
 *   KafkaTopicAssigner.generateAssignment            (reference: KafkaTopicAssigner.java:42-72,  "KTA")
 *     -> KafkaAssignmentStrategy.getRackAwareAssignment (KafkaAssignmentStrategy.java:40-63,      "KAS")
 *   as driven by the per-topic loop of KafkaAssignmentGenerator.printLeastDisruptiveReassignment
 *   (KafkaAssignmentGenerator.java:172-184, "KAG").
 *
 * Plain pointers and sizes only; no torch / C++ types. A Java maintainer binds these through JNI
 * (see INTEGRATION.md for the stub), a C++ host through kassign_host.hpp, Python through ctypes.
 *
 * The reference's per-topic method becomes a BATCH call: one ka_solve() == the whole KAG:173-184 loop
 * (T topics in order through ONE Context); a batch of 1 == one generateAssignment() call.
 *
 * All compute runs in hand-written sm_90a CUDA kernels. There is NO CPU fallback: without a usable
 * CUDA device ka_ctx_create() returns NULL and every entry point fails with KA_ERR_NO_DEVICE.
 */
#ifndef KASSIGN_H
#define KASSIGN_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* One ka_ctx == one `KafkaTopicAssigner` instance == one `KafkaAssignmentStrategy.Context`
 * (KTA:19-23, KAS:360-369): it owns the cross-topic leader-preference counters counter[broker][slot],
 * keyed by BROKER ID (so successive calls may use different broker sets, as the reference's tests do),
 * plus the device scratch. One in-flight call per ctx (the reference is single-threaded, KAS:361-368); different
 * ctxs may be used at the same time, from different host threads, and may have asynchronous calls in flight at once.
 * A call that takes a `stream` reads its device inputs, and writes its device outputs, in that stream's order: it sees
 * whatever was enqueued on `stream` before it, and work enqueued on `stream` after it sees its outputs.
 * A host call sees every earlier call of the same ctx: ka_ctx_get_counters, ka_ctx_set_counters, ka_ctx_reset,
 * ka_ctx_set_brokers, the host-buffer solves (ka_solve, ka_solve_dense and their _json forms), ka_last_status and
 * ka_ctx_destroy first wait on the host for the ctx's earlier asynchronous calls to finish on their streams, so a read sees
 * what they wrote and a write cannot reach what they still read. This rule adds no host wait to the calls that take a
 * `stream`. */
typedef struct ka_ctx ka_ctx;

/* Error report. `code` > 0 are the reference's exceptions; `topic_index` is the LOWEST failing topic in
 * loop order (KAG:173 aborts at the first throw) and, inside it, the first failure in the reference's own
 * evaluation order. After code != 0 the ctx counters are undefined (the reference process would be dead). */
typedef struct ka_status {
    int32_t code;
    int32_t topic_index; /* -1 when not topic-specific */
    int32_t partition;   /* partition id (from part_id, or the ordinal when part_id == NULL); -1 if n/a */
    int32_t a;           /* operand 1 of the message (see codes) */
    int32_t b;           /* operand 2 */
} ka_status;

enum {
    KA_OK = 0,
    /* IllegalStateException "Topic T has partition P with unexpected replication factor K"  KTA:58-60; a=K */
    KA_ERR_RF_MISMATCH = 1,
    /* IllegalStateException "Topic T does not have a positive replication factor!"           KTA:65-66 */
    KA_ERR_RF_NOT_POSITIVE = 2,
    /* IllegalStateException "Topic T has a higher replication factor (RF) than available brokers!" KTA:67-69; a=RF */
    KA_ERR_RF_GT_BROKERS = 3,
    /* IllegalStateException "Partition P could not be fully assigned!"                        KAS:183-184 */
    KA_ERR_UNASSIGNABLE = 4,
    /* ArrayIndexOutOfBoundsException from getNodeProcessingOrder when topic.hashCode()==Integer.MIN_VALUE
     * (Math.abs stays negative)                                                               KAS:190-192; a=index, b=length */
    KA_ERR_HASH_INDEX = 5,
    /* library-side failures (no reference counterpart) */
    KA_ERR_BAD_ARG = -1,
    KA_ERR_CUDA = -2,
    KA_ERR_NO_DEVICE = -3,
    KA_ERR_LIMIT = -4 /* a size beyond what the kernels' shared-memory layout supports; a=offending value */
};

/* ---- lifetime ---------------------------------------------------------------------------------- */

/* `new KafkaTopicAssigner()` (KTA:21-23). device = CUDA ordinal. NULL if no CUDA device/driver. */
ka_ctx* ka_ctx_create(int32_t device);
/* Waits for a pending asynchronous call of the ctx (on the stream it was enqueued on, which must still exist), then frees
 * the ctx. The call's outputs are complete in its stream's order. */
void ka_ctx_destroy(ka_ctx* ctx);
/* Drop all counters: a fresh Context (KAS:365-368). */
int32_t ka_ctx_reset(ka_ctx* ctx);

/* ---- the broker table ---------------------------------------------------------------------------
 * `brokers` + `rackAssignment` of generateAssignment (KTA:43-44) — the same for every topic of a run
 * (KAG:150-151,175-176) — uploaded once per run.
 *   broker_id[N]   strictly ascending live broker ids (the TreeMap order of KAS:78)
 *   broker_rack[N] dense rack index per broker, 0 <= idx < N. Brokers without a rack get an index no
 *                  other broker uses unless their decimal id equals a real rack's NAME (the string-key
 *                  quirk of KAS:82-94) — ka_rack_indices() below does that mapping from strings.
 * Counters of brokers that leave the set are retained (keyed by id) and come back if the id returns. */
int32_t ka_ctx_set_brokers(ka_ctx* ctx, int32_t N, const int32_t* broker_id, const int32_t* broker_rack);

/* Helper for the string side of KAS:81-94: rack_name[i] (NUL-terminated UTF-8, or NULL = "no rack
 * defined for this broker") -> dense indices with the id.toString() fallback and its collision quirk. */
int32_t ka_rack_indices(int32_t N, const int32_t* broker_id, const char* const* rack_name, int32_t* broker_rack);

/* java.lang.String.hashCode of a UTF-8 encoded topic name (UTF-16 code units, int32 wrap) — KAS:190. */
int32_t ka_java_string_hash(const char* utf8);

/* The name rule of every _json entry point: the device emitters copy topic names verbatim, so a name holding a character
 * that org.json 20131018's JSONObject.quote() rewrites is refused (KA_ERR_BAD_ARG with a = that character's code point; take
 * a host emitter instead). Over the len bytes of the UTF-8 name (NULs included), the first of: a byte below 0x20, '"', '\\'
 * or '/' (org.json escapes '/' only after '<'; every '/' is refused); the UTF-8 form of U+0080..U+009F (C2 80 .. C2 9F) or
 * of U+2000..U+20FF (E2 80 80 .. E2 83 BF). Returns its code point, or -1 when the name passes. Host only; needs no device. */
int32_t ka_json_name_refused(const char* name, int64_t len);

/* ---- the solve ----------------------------------------------------------------------------------
 * General (ragged) form, HOST buffers; copies in, runs the kernels, copies out, synchronises.
 *   T                topics, solved in index order through this ctx (KAG:173)
 *   topic_hash[T]    String.hashCode of each topic name
 *   part_off[T+1]    partitions of topic t are rows part_off[t] .. part_off[t+1]-1
 *   part_id[ΣP]      partition ids, ascending within a topic (TreeMap order, KAS:107-110); NULL = 0..P-1.
 *                    Only used to report ka_status.partition (and printed by ka_solve_json); the solver works on ordinals.
 *   rep_off[ΣP+1]    current replica list of row g is cur_broker[rep_off[g] .. rep_off[g+1]-1] (leader first)
 *   desired_rf       --desired_replication_factor; -1 = keep (KTA:49,55-61)
 *   out_stride       slots per output row; must be >= max(list length, target RF) over all rows
 *   out_len[ΣP]      length of each new replica list (may be NULL)
 *   out_broker[ΣP*out_stride]  new replica lists, leader first, in row order; unused slots = -1
 * Returns st->code. */
int32_t ka_solve(ka_ctx* ctx, int32_t T, const int32_t* topic_hash, const int64_t* part_off,
                 const int32_t* part_id, const int64_t* rep_off, const int32_t* cur_broker,
                 int32_t desired_rf, int32_t out_stride, int32_t* out_len, int32_t* out_broker,
                 ka_status* st);

/* Dense form (every topic P partitions 0..P-1, every list RF long): cur[T][P][RF] -> out[T][P][out_stride]. */
int32_t ka_solve_dense(ka_ctx* ctx, int32_t T, const int32_t* topic_hash, int32_t P, int32_t RF,
                       const int32_t* cur_broker, int32_t desired_rf, int32_t out_stride,
                       int32_t* out_len, int32_t* out_broker, ka_status* st);

/* Dense solve + the reference's JSON emitter (KAG:169-186) in one call: the rows never leave the device, only the TEXT
 *   {"partitions":[{"partition":p,"replicas":[..],"topic":"name"},...],"version":1}
 * crosses PCIe, streamed block by block while later topic blocks are still being ordered. names = the T topic names
 * concatenated (UTF-8; a name ka_json_name_refused refuses gives KA_ERR_BAD_ARG with a = the refused character's code
 * point: use the host emitter), name_off[T+1] their offsets;
 * json = host buffer of json_cap bytes (pinned for full PCIe speed; KA_ERR_LIMIT if too small: 64 + sum over rows of
 * (50 + 12*out_stride + name length) always suffices); *json_bytes = length of the text (not NUL-terminated).
 * A topic's exception wins over KA_ERR_LIMIT: when a topic fails, *st is what ka_solve_dense reports, whatever json_cap is, and
 * *json_bytes = 0. */
int32_t ka_solve_dense_json(ka_ctx* ctx, int32_t T, const int32_t* topic_hash, int32_t P, int32_t RF,
                            const int32_t* cur_broker, int32_t desired_rf, const char* names, const int64_t* name_off,
                            char* json, int64_t json_cap, int64_t* json_bytes, ka_status* st);

/* General (ragged) solve + the reference's JSON emitter: the inputs of ka_solve (part_id, NULL = 0..P-1, is what the text
 * prints as "partition"), the name slab and output contract of ka_solve_dense_json. The row stride is internal:
 * max(longest current list, desired_rf, 1). The text is cut into fragments of a fixed number of rows, each streamed out as
 * soon as it is built. json_cap = 64 + sum over rows of (50 + 12*stride + name length of the row's topic) always suffices
 * (it holds for any int32 partition id); KA_ERR_LIMIT if json_cap is too small. A run without rows (T == 0, or only empty
 * topics under a desired_rf) gives {"partitions":[],"version":1}. A name ka_json_name_refused refuses gives KA_ERR_BAD_ARG
 * with a = the refused character's code point before anything is solved (counters untouched). On any error *json_bytes = 0
 * and *st is what ka_solve reports for the same input; the ctx counters afterwards equal those after ka_solve. */
int32_t ka_solve_json(ka_ctx* ctx, int32_t T, const int32_t* topic_hash, const int64_t* part_off, const int32_t* part_id,
                      const int64_t* rep_off, const int32_t* cur_broker, int32_t desired_rf,
                      const char* names, const int64_t* name_off, char* json, int64_t json_cap,
                      int64_t* json_bytes, ka_status* st);

/* Dense form on DEVICE buffers (d_* are device pointers on the ctx's device; d_out_len may be NULL),
 * enqueued on `stream` (a cudaStream_t, NULL = the legacy default stream) — inputs already resident in
 * HBM, outputs left in HBM. If st != NULL the call synchronises the stream and fills *st; with
 * st == NULL it is fully asynchronous and the status is fetched later with ka_last_status(); work enqueued on `stream`
 * after the call may read the outputs without any host synchronisation. */
int32_t ka_solve_dense_device(ka_ctx* ctx, int32_t T, const int32_t* d_topic_hash, int32_t P, int32_t RF,
                              const int32_t* d_cur_broker, int32_t desired_rf, int32_t out_stride,
                              int32_t* d_out_len, int32_t* d_out_broker, void* stream, ka_status* st);

/* The dense problem of ka_solve_dense_device, solved against K candidate broker tables, each on a FRESH Context
 * (all counters zero) — K independent runs of the reference tool over one cluster (KAG:172, one assigner per run), e.g. the
 * broker sets of a decommission sweep. The candidates run side by side inside every kernel: the number of kernel launches
 * does not depend on K.
 *   cand_off[K+1]      host; table k is broker_id/broker_rack[cand_off[k] .. cand_off[k+1]-1]
 *   broker_id, broker_rack   host; per table, exactly what ka_ctx_set_brokers takes (ids strictly ascending, rack index)
 *   d_topic_hash, d_cur_broker   device, shared by all candidates
 *   d_out_broker       device [K][T*P][out_stride]; d_out_len device [K][T*P] or NULL
 *   st[K]              host, required; st[k] is candidate k's status
 * Candidate k gives exactly what ka_ctx_create -> ka_ctx_set_brokers(table k) -> ka_solve_dense_device gives: the same rows,
 * out_len and status fields. The rows of a failed candidate are unspecified; a failing candidate changes nothing of another.
 * Limits, checked before anything is enqueued: K <= 128 and out_stride <= 3 (else KA_ERR_LIMIT); out_stride >=
 * max(RF, desired_rf) (else KA_ERR_BAD_ARG); every table as ka_ctx_set_brokers checks it (same code). K == 0 or T == 0:
 * KA_OK, nothing written.
 * Synchronises `stream` before returning. Returns KA_OK when every candidate solved, else st[k].code of the lowest failing k;
 * library-side failures (bad argument, limit, CUDA) are returned directly and written to every st[k].
 * Does not read or change ctx's own Context, broker table, parked counters or topic_base. */
int32_t ka_solve_dense_candidates_device(ka_ctx* ctx, int32_t K, const int32_t* cand_off, const int32_t* broker_id,
                                         const int32_t* broker_rack, int32_t T, const int32_t* d_topic_hash, int32_t P,
                                         int32_t RF, const int32_t* d_cur_broker, int32_t desired_rf, int32_t out_stride,
                                         int32_t* d_out_len, int32_t* d_out_broker, void* stream, ka_status* st);

/* The general (ragged) problem of ka_solve, in HOST buffers, solved against K candidate broker tables, each on a FRESH
 * Context: K runs of the reference tool over one real cluster, e.g. the broker sets of a decommission sweep.
 *   cand_off, broker_id, broker_rack   the candidate tables, as ka_solve_dense_candidates_device takes them
 *   T .. desired_rf    the inputs of ka_solve (part_id, NULL = 0..P-1, is only used for ka_status.partition)
 *   out_broker[K][ΣP][out_stride], out_len[K][ΣP] (or NULL)   host; candidate k's rows and list lengths
 *   st[K]              host, required; st[k] is candidate k's status
 * Candidate k gives exactly what ka_ctx_create -> ka_ctx_set_brokers(table k) -> ka_solve(same inputs, out_stride) gives: the
 * same rows, out_len and status fields (partition mapped through part_id). The rows of a failed candidate are unspecified; a
 * failing candidate changes nothing of another. The problem's inputs are copied to the device once and shared by all
 * candidates; the number of kernel launches does not depend on K.
 * Limits, checked before anything is enqueued: K <= 128, out_stride <= 3 and K * ΣP < 2^31 (else KA_ERR_LIMIT); out_stride >=
 * max(longest current list, desired_rf) (else KA_ERR_BAD_ARG), so that every accepted input is one ka_solve accepts for
 * every table; every table as ka_ctx_set_brokers checks it and every offset array as ka_solve checks it (same status).
 * K == 0 or T == 0: KA_OK, nothing written. Topics without partitions are solved (and may fail) as ka_solve solves them.
 * Synchronous. Returns KA_OK when every candidate solved, else st[k].code of the lowest failing k; library-side failures are
 * returned directly and written to every st[k]. Does not read or change ctx's own Context, broker table, parked counters,
 * topic_base or staged block. */
int32_t ka_solve_candidates(ka_ctx* ctx, int32_t K, const int32_t* cand_off, const int32_t* broker_id,
                            const int32_t* broker_rack, int32_t T, const int32_t* topic_hash, const int64_t* part_off,
                            const int32_t* part_id, const int64_t* rep_off, const int32_t* cur_broker,
                            int32_t desired_rf, int32_t out_stride, int32_t* out_len, int32_t* out_broker,
                            ka_status* st);

/* A fleet of K independent clusters, each solved against its OWN broker table on a FRESH Context, in one call: K runs of the
 * reference tool, one per cluster (a fleet-wide host retirement or OS roll, a rack move that touches several clusters). The
 * clusters run side by side inside every kernel; the number of kernel launches does not depend on K, and the call takes about
 * as long as its longest cluster's leader-order chain.
 *   cand_off, broker_id, broker_rack   table k is cluster k's, as ka_solve_candidates takes the candidate tables
 *   topic_off[K+1]     host; cluster k is topics topic_off[k] .. topic_off[k+1]-1 of the inputs below
 *   desired_rf[K]      host; cluster k's --desired_replication_factor, or NULL = -1 for every cluster
 *   topic_hash .. cur_broker   ONE ragged layout (as ka_solve takes it) over all ΣT topics and ΣP rows, host
 *   out_broker[ΣP][out_stride], out_len[ΣP] (or NULL)   host; every row at its place in the layout
 *   st[K]              host, required; st[k] is cluster k's status
 * Cluster k's rows, out_len entries and st[k] are exactly what ka_ctx_create -> ka_ctx_set_brokers(table k) -> ka_solve(its
 * topics, with part_off / rep_off rebased to 0, desired_rf[k], out_stride) gives: topic_index counts from the cluster's first
 * topic, partition is mapped through part_id. A failing cluster changes nothing of another; its rows are unspecified. What
 * ka_solve would report for a cluster's slice (malformed offsets inside it, lists longer than out_stride, a target RF in
 * (out_stride, N], a table beyond the level plan's broker limit, the five reference exceptions) is that cluster's status,
 * and the others still solve.
 * Checked for the whole call (the code in every st[k], and returned): K <= 128 and out_stride <= 3 (else KA_ERR_LIMIT);
 * out_stride >= 1; every table as ka_ctx_set_brokers checks it (same code); topic_off non-decreasing from 0, and part_off at
 * every cluster's first topic and rep_off at its first row non-decreasing from 0 (else KA_ERR_BAD_ARG); ΣP < 2^31 (else
 * KA_ERR_LIMIT). One plan serves the call, sized from its largest table and largest topic: if that plan exceeds shared memory
 * where no cluster's own does, every st[k] is KA_ERR_LIMIT. K == 0: KA_OK, nothing written.
 * Synchronous. Returns KA_OK when every cluster solved, else st[k].code of the lowest failing k. Does not read or change ctx's
 * own Context, broker table, parked counters, topic_base or staged block. */
int32_t ka_solve_clusters(ka_ctx* ctx, int32_t K, const int32_t* cand_off, const int32_t* broker_id,
                          const int32_t* broker_rack, const int32_t* topic_off, const int32_t* desired_rf,
                          const int32_t* topic_hash, const int64_t* part_off, const int32_t* part_id,
                          const int64_t* rep_off, const int32_t* cur_broker, int32_t out_stride,
                          int32_t* out_len, int32_t* out_broker, ka_status* st);

/* The fleet of ka_solve_clusters, each cluster's rows turned into that cluster's reassignment JSON on the device: one document
 * per cluster, and only the text crosses PCIe.
 *   K .. cur_broker    the fleet inputs of ka_solve_clusters (no out_stride: the stride is internal, see below)
 *   names, name_off    the names of all ΣT topics in input order, as ka_solve_json takes them (name_off[ΣT+1])
 *   json               host buffer of json_cap bytes (pinned for full PCIe speed)
 *   json_off[K+1]      host; cluster k's document is json[json_off[k] .. json_off[k+1]), back to back in cluster order, not
 *                      NUL-terminated; json_off[0] = 0, and a cluster that failed has an empty range
 *   st[K]              host, required; st[k] is cluster k's status
 * Cluster k's text and st[k] are exactly what ka_ctx_create -> ka_ctx_set_brokers(table k) -> ka_solve_json(its topics, with
 * part_off / rep_off rebased to 0 and its names, desired_rf[k]) gives: topic_index counts from the cluster's first topic,
 * partition is mapped through part_id. A cluster without topics, or with only empty topics under a desired RF, gets
 * {"partitions":[],"version":1}. Per cluster, in ka_solve_json's order: the sizing scan and capacity checks of ka_solve_clusters;
 * a name ka_json_name_refused refuses (KA_ERR_BAD_ARG, a = its code point); the 32-bit fragment limit of ka_solve_json; the
 * cluster's own plan; the five reference exceptions. A cluster that fails any of them has no text, and the others still solve.
 * Stride: cluster k's width is max(longest current list, desired_rf[k], 1), and the call runs at the largest width among the
 * clusters it solves. The batched chains take rows of at most 3, so a cluster wider than 3 gets KA_ERR_LIMIT with a = its
 * width (the one difference from ka_solve_json, which solves widths 4..8 through its fused chain).
 * Checked for the whole call (the code in every st[k], and returned): what ka_solve_clusters checks for the whole call (K,
 * tables, cluster boundaries, ΣP < 2^31); names or name_off NULL when ΣT > 0, json or json_off NULL, json_cap < 0
 * (KA_ERR_BAD_ARG); a plan or fragment size of the whole call that fails where no cluster's own does (KA_ERR_LIMIT).
 * Buffer: sum over clusters k of (64 + sum over cluster k's rows of (50 + 12 * width k + name length of the row's topic))
 * always suffices. If json_cap is too small, every cluster that solved gets KA_ERR_LIMIT with a = min(json_cap, INT_MAX), a
 * failed cluster keeps its status, and every json_off[k] is 0. K == 0: KA_OK, json_off[0] = 0.
 * Synchronous. Returns KA_OK when every cluster solved, else st[k].code of the lowest failing k. The number of kernel launches
 * depends on ΣP and not on K. Does not read or change ctx's own Context, broker table, parked counters, topic_base or staged
 * block. */
int32_t ka_solve_clusters_json(ka_ctx* ctx, int32_t K, const int32_t* cand_off, const int32_t* broker_id,
                               const int32_t* broker_rack, const int32_t* topic_off, const int32_t* desired_rf,
                               const int32_t* topic_hash, const int64_t* part_off, const int32_t* part_id,
                               const int64_t* rep_off, const int32_t* cur_broker, const char* names, const int64_t* name_off,
                               char* json, int64_t json_cap, int64_t* json_off, ka_status* st);

/* What a candidate's rows change against the current lists, and how they spread over its brokers. Every field is int64, so
 * the layout has no padding. Position counts: a duplicate id in a current list, or a current broker the table lacks, needs
 * no special case. w[g] is the weight of row g (1 without weights); the rows_* and leaders_changed fields count rows. */
typedef struct ka_move_summary {
    int64_t rows_changed;       /* rows whose new list differs from the current one (length or any position) */
    int64_t rows_moved;         /* rows with at least one added or dropped replica */
    int64_t leaders_changed;    /* rows whose current list is empty or whose first broker changed */
    int64_t replicas_added;     /* sum of w[g] x (positions of the new list whose broker is not in the current list) */
    int64_t replicas_dropped;   /* sum of w[g] x (positions of the current list whose broker is not in the new list) */
    int64_t max_broker_in;      /* largest per-broker sum of added replicas (the receiving bottleneck) ... */
    int64_t max_broker_in_id;   /* ... and that broker's id (lowest id on ties; -1 when no broker receives anything) */
    int64_t max_broker_replicas, min_broker_replicas;   /* sum of w over the replicas each live broker holds after the move */
    int64_t max_broker_leaders, min_broker_leaders;     /* sum of w over the rows each live broker leads after the move */
} ka_move_summary;

/* ka_solve_candidates, scored on the device: a few numbers per candidate instead of K copies of the rows, to choose between
 * the broker sets of a sweep.
 *   K .. out_stride     exactly as ka_solve_candidates takes them
 *   part_weight[ΣP]     host, >= 0 per row (e.g. the partition's size in bytes), or NULL = 1 per row
 *   summary[K]          host, required; summary[k] is a function of candidate k's rows and the current lists only
 *   broker_replicas, broker_leaders, broker_in   host [cand_off[K]] each, or NULL: entry cand_off[k] + i belongs to broker
 *                       broker_id[cand_off[k] + i] (replicas held, rows led and replicas added, each weighted)
 *   out_len, out_broker as ka_solve_candidates takes them, or out_broker == NULL: the rows stay on the device
 *   st[K]               host, required
 * st[k], the return code and (when out_broker is given) the rows are exactly what ka_solve_candidates gives for the same inputs.
 * A failed candidate, and every candidate when T == 0, gets a zero summary with max_broker_in_id = -1 and zero per-broker
 * entries. Checked after every check of ka_solve_candidates and before anything is enqueued: a negative weight gives
 * KA_ERR_BAD_ARG, 3 x (sum of weights) > INT64_MAX gives KA_ERR_LIMIT. Adds a fixed number of kernel launches, independent
 * of K. Synchronous. Does not read or change ctx's own Context, broker table, parked counters, topic_base or staged block. */
int32_t ka_score_candidates(ka_ctx* ctx, int32_t K, const int32_t* cand_off, const int32_t* broker_id,
                            const int32_t* broker_rack, int32_t T, const int32_t* topic_hash, const int64_t* part_off,
                            const int32_t* part_id, const int64_t* rep_off, const int32_t* cur_broker, int32_t desired_rf,
                            int32_t out_stride, const int64_t* part_weight, ka_move_summary* summary,
                            int64_t* broker_replicas, int64_t* broker_leaders, int64_t* broker_in,
                            int32_t* out_len, int32_t* out_broker, ka_status* st);

/* ka_solve_clusters, scored on the device: per cluster of a fleet, how much data its new assignment moves, which broker
 * receives the most and how evenly it leaves replicas and leaders, before any of the K documents goes to the cluster.
 *   K .. out_stride     exactly as ka_solve_clusters takes them
 *   part_weight[ΣP]     host, >= 0 per row of the shared layout (e.g. the partition's size in bytes), or NULL = 1 per row
 *   summary[K]          host, required; summary[k] is a function of cluster k's rows and current lists only
 *   broker_replicas, broker_leaders, broker_in   host [cand_off[K]] each, or NULL: entry cand_off[k] + i belongs to broker
 *                       broker_id[cand_off[k] + i] of cluster k (replicas held, rows led and replicas added, each weighted)
 *   out_len, out_broker as ka_solve_clusters takes them, or out_broker == NULL: the rows stay on the device
 *   st[K]               host, required
 * st[k], the return code and (when out_broker is given) the rows are exactly what ka_solve_clusters gives for the same inputs.
 * A cluster that failed (refused by the checks of its slice or its own plan, or one of the five reference exceptions) gets a
 * zero summary with max_broker_in_id = -1 and zero per-broker entries, and so does a cluster that solved without rows. A
 * call refused as a whole writes zero summaries, and zero per-broker entries once the tables pass ka_ctx_set_brokers' checks.
 * Checked after every check of ka_solve_clusters and before anything is enqueued, over all ΣP rows, when some cluster is
 * left to solve: a negative weight gives KA_ERR_BAD_ARG, 3 x (sum of weights) > INT64_MAX gives KA_ERR_LIMIT, in every st[k].
 * Adds two kernel launches to those of ka_solve_clusters, whatever K is. Synchronous. Does not read or change ctx's own
 * Context, broker table, parked counters, topic_base or staged block. */
int32_t ka_score_clusters(ka_ctx* ctx, int32_t K, const int32_t* cand_off, const int32_t* broker_id,
                          const int32_t* broker_rack, const int32_t* topic_off, const int32_t* desired_rf,
                          const int32_t* topic_hash, const int64_t* part_off, const int32_t* part_id,
                          const int64_t* rep_off, const int32_t* cur_broker, int32_t out_stride,
                          const int64_t* part_weight, ka_move_summary* summary,
                          int64_t* broker_replicas, int64_t* broker_leaders, int64_t* broker_in,
                          int32_t* out_len, int32_t* out_broker, ka_status* st);

/* One wave of a reassignment cut into waves by ka_plan_waves. Every field is int64, so the layout has no padding. */
typedef struct ka_wave_summary {
    int64_t rows;               /* rows placed in the wave */
    int64_t rows_moved;         /* of them, rows with at least one receiver */
    int64_t replicas_added;     /* sum of w[g] x receivers */
    int64_t max_broker_in;      /* largest per-broker incoming sum in the wave ... */
    int64_t max_broker_in_id;   /* ... its broker id (lowest id on ties, -1 when nothing is added) */
} ka_wave_summary;

/* A reassignment cut into waves, consecutive documents in which no broker receives more than a budget: what an operator runs
 * one after the other instead of starting every new replica of a cluster at once.
 *   Q                  rows; row g's current list is cur_broker[rep_off[g] .. rep_off[g + 1]) (rep_off[Q+1], host)
 *   new_len[Q], new_broker[Q * stride]   host; the proposed lists, laid out as ka_solve's out_len / out_broker (its rows go in
 *                      unchanged); 1 <= stride <= 8
 *   part_weight[Q]     host, >= 0 per row (e.g. the partition's size in bytes), or NULL = 1 per row
 *   max_broker_in      the budget B >= 1
 *   wave[Q]            host, or NULL; the wave of every row (0 for a row that did not change)
 *   n_waves            host, required; *n_waves = W, the number of waves
 *   summary[summary_cap]   host; the first min(W, summary_cap) waves' summaries (NULL is allowed when summary_cap == 0)
 * The rule, over the broker table of ka_ctx_set_brokers. A row is CHANGED when its new list differs from the current one in
 * length or in any position (ka_move_summary's rows_changed); its RECEIVERS are the positions of the new list whose broker the
 * current list does not hold (ka_move_summary's replicas_added counts them). Each broker b of the table starts with
 * open[b] = 1, load[b] = 0, and the rows are taken in input order (permute the input to move some rows first):
 *   an unchanged row gets wave 0 and a changed row without receivers wave 1; otherwise, with w = w[g],
 *   wave[g] = max over its receivers b of (open[b] if load[b] == 0 or load[b] + w <= B, else open[b] + 1), and then every
 *   receiver b with wave[g] > open[b] gets open[b] = wave[g], load[b] = w, every other receiver load[b] += w.
 * So the waves are 1..W, none empty (W = 0 when no row changed); in every wave every broker receives at most B, unless a single
 * row heavier than B is its only incoming row of nonzero weight there; with B >= the sum of the weights everything is in wave 1. Under
 * this rule (KA_WAVE_GREEDY, a Context's default) a broker's waves only move forward (two words of state per broker): this is
 * a greedy rule, not an optimal packing — a later row never goes back to fill an earlier wave.
 * FIRST FIT (KA_WAVE_FIRST_FIT, chosen with ka_ctx_set_wave_rule) puts each row in the earliest wave where its receivers still
 * have room. Every (broker, wave) pair starts with load[b][v] = 0; unchanged rows and changed rows without receivers are as
 * above; any other row g takes wave[g] = the smallest v >= 1 in which every receiver b has load[b][v] == 0 or
 * load[b][v] + w <= B, then load[b][v] += w for every receiver. A broker's waves no longer only move forward: a later row fills
 * an earlier wave wherever every one of its receivers has room there. Every budget above holds exactly as under the greedy rule;
 * no wave is empty (a row takes wave v > 1 only when wave v - 1 is refused by a bucket with nonzero load), so W <= the changed
 * rows and every bound of the document calls holds unchanged; where no broker receives two moved rows the plan equals the
 * greedy one. With M the rows with receivers and R_b the moved rows b receives, W <= Wb = min(M, 1 + max over those rows of
 * the sum over their receivers of (R_b - 1)): a wave below a row's is refused only by a bucket holding an earlier row that
 * shares a receiver, and b has at most R_b - 1 of them. The device keeps a load table of Wb x N int64 words: after the row
 * errors, Wb x N x 8 > 2^30 bytes gives KA_ERR_LIMIT with a = Wb, before the plan runs. First fit adds 3 kernel launches and
 * one synchronisation (the bound, read back to size the table), whatever Q and W are.
 * Checks, in this order, before anything is enqueued: st NULL: KA_ERR_BAD_ARG (nothing written); ctx NULL: KA_ERR_NO_DEVICE;
 * Q < 0, stride < 1, n_waves NULL, summary_cap < 0, summary NULL with summary_cap > 0, max_broker_in < 1, or rep_off not
 * non-decreasing from 0 (or a needed array NULL): KA_ERR_BAD_ARG; stride > 8 or Q >= 2^31: KA_ERR_LIMIT; a new_len outside
 * [0, stride]: KA_ERR_BAD_ARG with a = the lowest such row; a negative weight: KA_ERR_BAD_ARG; 8 x (sum of weights) > INT64_MAX:
 * KA_ERR_LIMIT. On the device, the lowest failing row wins: a new list naming a broker twice, or a receiver the table lacks,
 * gives KA_ERR_BAD_ARG with a = the row and b = the broker id at the first such position of its list. On any error *n_waves = 0
 * and wave / summary are unspecified. Q == 0: KA_OK, W = 0. Duplicate or unknown ids in a current list need no special case.
 * Synchronous; adds a fixed number of kernel launches, whatever Q and W are. Follows the Context's wave rule
 * (ka_ctx_set_wave_rule); does not read or change the Context counters, parked counters, topic_base, the staged block, or the
 * last order / stage plans and timings. */
int32_t ka_plan_waves(ka_ctx* ctx, int64_t Q, const int64_t* rep_off, const int32_t* cur_broker, int32_t stride,
                      const int32_t* new_len, const int32_t* new_broker, const int64_t* part_weight, int64_t max_broker_in,
                      int32_t* wave, int32_t* n_waves, ka_wave_summary* summary, int32_t summary_cap, ka_status* st);

/* The wave rule every plan call of this Context follows: ka_plan_waves, ka_plan_waves_send and their _json, _json_parts and
 * _json_parts_rollback forms. Their checks, error codes and outputs keep their contracts under either rule; only wave[] (and
 * so W, the summaries and the documents) changes. Configuration like ka_ctx_set_timing: ka_ctx_reset leaves it alone. */
enum {
    KA_WAVE_GREEDY = 0,      /* the default: a broker's waves only move forward (ka_plan_waves, ka_plan_waves_send) */
    KA_WAVE_FIRST_FIT = 1    /* each row in the earliest wave where its receivers and its sender still have room */
};
/* KA_OK; any other rule: KA_ERR_BAD_ARG (the rule stays); ctx NULL: KA_ERR_NO_DEVICE. */
int32_t ka_ctx_set_wave_rule(ka_ctx* ctx, int32_t rule);
/* The Context's wave rule; ctx NULL: KA_ERR_NO_DEVICE. */
int32_t ka_ctx_wave_rule(ka_ctx* ctx);

/* The PART CAPS every _parts call of this Context follows: ka_plan_waves_json_parts, ka_plan_waves_send_json_parts and their
 * _rollback forms. The parts of a wave run one after the other, so one part is everything in flight at a time; the caps bound
 * it beside the byte limit L of those calls:
 *   max_part_rows = Lr   the most rows one part holds (0: no row cap)
 *   max_part_in = Lx     the most data one part moves (0: no data cap): with a_g = w[g] x the receivers of row g, exactly what
 *                        ka_wave_summary.replicas_added adds for the row (0 for a row that only reorders, w = 1 without
 *                        weights), a part's rows hold sum(a) <= Lx unless the part is a single row
 * The rule. Within one wave, rows i..j-1 (input order) make a part iff every byte condition of the call holds (S, and R on the
 * rollback side), j - i <= Lr when Lr is set, and sum over i..j-1 of a <= Lx or j - i == 1 when Lx is set. Every condition is
 * monotone in j, so the greedy cut stays unique, and no two consecutive parts of a wave could be merged under all of them. A
 * row with a_g > Lx makes a part of its own, as a row heavier than max_broker_in has a wave to itself; it is not an error, and
 * the caps add no error code (sum(a) <= 8 x the sum of the weights <= INT64_MAX is checked already). Any subset of a wave keeps
 * every budget of that wave, so the plan, wave[], W and the summaries are those of the uncapped call; D <= the changed rows <=
 * Q still holds, so doc_off[Q+1], doc_wave[Q] and the json_cap / back_cap bounds are unchanged. With both caps 0 every output
 * is byte for byte that of a Context that never set them. The caps add no kernel launch and no synchronisation.
 * ka_plan_waves(_send)(_json) make no parts and ignore the caps. Configuration like the wave rule: ka_ctx_reset leaves it alone.
 * KA_OK; a negative value: KA_ERR_BAD_ARG (the caps stay as they were); ctx NULL: KA_ERR_NO_DEVICE. */
int32_t ka_ctx_set_part_caps(ka_ctx* ctx, int64_t max_part_rows, int64_t max_part_in);
/* The Context's part caps into *max_part_rows and *max_part_in (0 = no cap); ctx NULL: KA_ERR_NO_DEVICE; an output NULL:
 * KA_ERR_BAD_ARG. */
int32_t ka_ctx_part_caps(ka_ctx* ctx, int64_t* max_part_rows, int64_t* max_part_in);

/* ka_plan_waves + the documents it plans, built on the device: one reassignment JSON per wave, what an operator feeds
 * kafka-reassign-partitions one after the other. Only the text, the waves and the summaries cross PCIe.
 *   T, part_off[T+1], part_id (NULL = 0..P-1 per topic), names, name_off[T+1]   host; the ragged layout and the name slab
 *                      exactly as ka_solve_json takes them; Q = part_off[T] rows
 *   rep_off .. max_broker_in   exactly as ka_plan_waves takes them, over those Q rows
 *   wave, n_waves, summary, summary_cap   exactly as ka_plan_waves writes them: the same values for the same inputs
 *   json               host buffer of json_cap bytes (pinned for full PCIe speed)
 *   doc_off[Q+1]       host, required when Q > 0 (W never exceeds Q, so no second call is ever needed); entries 0..W are written,
 *                      doc_off[0] = 0
 * Document v, the one of wave v + 1, is json[doc_off[v] .. doc_off[v+1]): the documents lie back to back and are not
 * NUL-terminated. It is {"partitions":[ + the records of the rows with wave[g] == v + 1, in input row order, comma separated +
 * ],"version":1}, a record being byte for byte the one ka_solve_json prints for that row (its topic's name, its partition
 * through part_id, its new list). Unchanged rows (wave 0) are in no document, a changed row is in exactly one. W == 0 (nothing
 * changed, or Q == 0) gives no document: doc_off[0] = 0 (when doc_off is given), KA_OK.
 * json_cap = the sum over rows of (79 + 12*stride + name length of the row's topic) always suffices: the 50 + 12*stride + name
 * of a record of ka_solve_json, and the 29 bytes of a document's header and trailer charged to every row, because a wave has at
 * least one row.
 * Checks, in this order, before anything is enqueued: st NULL: KA_ERR_BAD_ARG (nothing written); ctx NULL: KA_ERR_NO_DEVICE;
 * everything ka_plan_waves checks, with its codes and operands (T < 0, or part_off NULL with T > 0, leaves no Q to check:
 * KA_ERR_BAD_ARG); then part_off not non-decreasing from 0, names or name_off NULL with T > 0, json NULL, json_cap < 0, or
 * doc_off NULL with Q > 0: KA_ERR_BAD_ARG; then a name ka_json_name_refused refuses: KA_ERR_BAD_ARG with a = the
 * refused character's code point (take ka_plan_waves and a host emitter instead). On the device the plan's own row errors
 * come first, with the code, a and b of ka_plan_waves; a text longer than json_cap gives KA_ERR_LIMIT with a = min(json_cap, INT_MAX). On any error *n_waves = 0 and
 * nothing else is specified.
 * Synchronous. The kernel launches it adds depend only on the bit length of W (one stable radix pass over the waves per 8
 * bits), not on Q or T. Follows the Context's wave rule (ka_ctx_set_wave_rule); does not read or change the Context counters, parked counters, topic_base, the staged block, or the
 * last order / stage plans and timings. */
int32_t ka_plan_waves_json(ka_ctx* ctx, int32_t T, const int64_t* part_off, const int32_t* part_id,
                           const int64_t* rep_off, const int32_t* cur_broker, int32_t stride,
                           const int32_t* new_len, const int32_t* new_broker, const int64_t* part_weight,
                           int64_t max_broker_in, const char* names, const int64_t* name_off,
                           char* json, int64_t json_cap, int64_t* doc_off,
                           int32_t* wave, int32_t* n_waves, ka_wave_summary* summary, int32_t summary_cap,
                           ka_status* st);

/* What the partitions' leaders send in one wave of ka_plan_waves_send, beside that wave's ka_wave_summary. */
typedef struct ka_wave_send_summary {
    int64_t max_broker_out;     /* largest per-broker outgoing sum in the wave ... */
    int64_t max_broker_out_id;  /* ... its broker id (lowest id on ties, -1 when nothing is sent) */
} ka_wave_send_summary;

/* ka_plan_waves with a sender budget as well: no broker SENDS more than max_broker_out = C per wave either. A new replica
 * fetches the whole partition from its leader, so a plan that caps only what each broker receives can still have one leader
 * (typically a drained broker) send to every receiver of the cluster in one wave; Kafka throttles both sides
 * (leader.replication.throttled.rate and follower.replication.throttled.rate) for this reason.
 *   Q .. max_broker_in  exactly as ka_plan_waves takes them
 *   n_send, send_id[n_send]   host; the SEND TABLE, strictly ascending ids (typically every broker of the cluster before an
 *                      exclusion: a drained broker sends but is not in the ctx's broker table); 0 <= n_send <= 65535
 *   max_broker_out     the sender budget C >= 1
 *   wave, n_waves, summary   as ka_plan_waves writes them, under the rule below
 *   send_summary[summary_cap]   host; the first min(W, summary_cap) waves' sender summaries, send_summary[v] beside summary[v]
 *                      (NULL is allowed when summary_cap == 0)
 * The rule is ka_plan_waves's with one more term and one more update per row with receivers. Its SENDER is the first broker of
 * its current list (the preferred leader, which leads the partition in a balanced cluster); a row whose current list is empty
 * has no sender. Each sender s of the send table starts with sopen[s] = 1, sload[s] = 0; a row of weight w with r receivers
 * sends a = w x r. wave[g] = the max of ka_plan_waves's receiver terms and, for its sender s, (sopen[s] if sload[s] == 0 or
 * sload[s] + a <= C, else sopen[s] + 1). Then the receivers update as in ka_plan_waves, and the sender likewise: wave[g] >
 * sopen[s] gives sopen[s] = wave[g], sload[s] = a, else sload[s] += a. Sending and receiving are separate budgets: a broker can
 * be the sender of one row and a receiver of another.
 * So in every wave every broker sends at most C, unless a single row with w x r > C is its only outgoing row of nonzero weight
 * there; every receive bound of ka_plan_waves still holds; the waves are still 1..W and none is empty (every wave value is some
 * broker's open or open + 1), so doc_off and the json_cap bound of ka_plan_waves_json hold unchanged. Like a receiver, a
 * leader's waves only move forward under the greedy rule: a row never goes to an earlier wave than its leader's open one.
 * Under KA_WAVE_FIRST_FIT the sender is one more bucket per wave: wave[g] = the smallest v >= 1 in which every receiver fits as
 * in ka_plan_waves and its sender s has sload[s][v] == 0 or sload[s][v] + a <= C; then sload[s][v] += a. Every bound above
 * holds; where no broker receives two moved rows and no sender sends two, the plan equals the greedy one. Wb adds
 * (S_s - 1) to each row's sum, S_s the moved rows s sends, and the load table is Wb x (N + n_send) words: Wb x (N + n_send) x
 * 8 > 2^30 gives KA_ERR_LIMIT with a = Wb. With C >= 8 x (sum of the
 * weights) no leader ever opens a wave, so a row's wave is the larger of ka_plan_waves's receiver terms and its leader's open
 * wave; where no leader has two moved rows, wave, W, summary and every document are exactly those of ka_plan_waves(_json).
 * Checks: everything ka_plan_waves checks, in its order, with its codes and operands; then max_broker_out < 1, n_send < 0,
 * send_id NULL with n_send > 0, send_id not strictly ascending, or send_summary NULL with summary_cap > 0: KA_ERR_BAD_ARG;
 * n_send > 65535: KA_ERR_LIMIT with a = n_send. On the device, the lowest failing row wins, over ka_plan_waves's row errors and
 * this one together: a row with receivers whose sender the send table lacks gives KA_ERR_BAD_ARG with a = the row and b = the
 * sender's id; within a row, the new-list errors come first. On any error *n_waves = 0 and nothing else is specified.
 * Synchronous; 9 kernel launches (ka_plan_waves's 7 and 2 over the sender buckets), whatever Q, W and n_send are, and the 3 of
 * first fit. Follows the Context's wave rule; does not read or change the Context counters, parked counters, topic_base, the staged block, or the last order / stage plans and timings. */
int32_t ka_plan_waves_send(ka_ctx* ctx, int64_t Q, const int64_t* rep_off, const int32_t* cur_broker, int32_t stride,
                           const int32_t* new_len, const int32_t* new_broker, const int64_t* part_weight, int64_t max_broker_in,
                           int32_t n_send, const int32_t* send_id, int64_t max_broker_out,
                           int32_t* wave, int32_t* n_waves, ka_wave_summary* summary, ka_wave_send_summary* send_summary,
                           int32_t summary_cap, ka_status* st);

/* ka_plan_waves_json under the rule of ka_plan_waves_send: the documents of its waves, built on the device.
 *   T .. max_broker_in, names .. summary   exactly as ka_plan_waves_json takes and writes them
 *   n_send, send_id, max_broker_out, send_summary   exactly as ka_plan_waves_send takes and writes them
 * Every wave is non-empty, so doc_off[Q+1] and the json_cap bound of ka_plan_waves_json hold unchanged.
 * Checks: everything ka_plan_waves_json checks, in its order; then the sender checks of ka_plan_waves_send. On the device the
 * row errors of ka_plan_waves_send come first; a text longer than json_cap gives KA_ERR_LIMIT with a = min(json_cap, INT_MAX).
 * Follows the Context's wave rule (ka_ctx_set_wave_rule). Synchronous; the launches of ka_plan_waves_send, then, when W > 0, 3 per 8 bits of W and 3 more. */
int32_t ka_plan_waves_send_json(ka_ctx* ctx, int32_t T, const int64_t* part_off, const int32_t* part_id,
                                const int64_t* rep_off, const int32_t* cur_broker, int32_t stride,
                                const int32_t* new_len, const int32_t* new_broker, const int64_t* part_weight,
                                int64_t max_broker_in, int32_t n_send, const int32_t* send_id, int64_t max_broker_out,
                                const char* names, const int64_t* name_off, char* json, int64_t json_cap, int64_t* doc_off,
                                int32_t* wave, int32_t* n_waves, ka_wave_summary* summary, ka_wave_send_summary* send_summary,
                                int32_t summary_cap, ka_status* st);

/* ka_plan_waves_json with every document under a size limit: each wave cut on the device into PARTS of at most L =
 * max_doc_bytes bytes, documents that run one after the other. Kafka 0.10's kafka-reassign-partitions writes a whole document
 * into one ZooKeeper znode, and ZooKeeper refuses znode data above jute.maxbuffer (0xfffff bytes by default): L = 1048575 gives
 * documents it accepts. Any subset of a wave keeps every receive (and send) budget of that wave, so cutting a wave weakens no
 * guarantee of the plan.
 *   T .. json_cap, wave, n_waves, summary, summary_cap   exactly as ka_plan_waves_json takes and writes them: wave, W and the
 *                      summaries are those of ka_plan_waves for the same inputs
 *   max_doc_bytes      the limit L >= 1
 *   doc_off[Q+1]       host, required when Q > 0; entries 0..D are written, doc_off[0] = 0
 *   doc_wave[Q]        host, required when Q > 0; doc_wave[d] = the wave (1..W) of part d, for d < D
 *   n_docs             host, required when Q > 0; *n_docs = D, the number of parts
 * The rule. Take the rows of wave v in input row order, and let b_i be the byte length of row i's record: exactly the record
 * ka_solve_json prints, without its comma. A part is a run of consecutive rows of one wave; its document is {"partitions":[ +
 * the records, comma separated, + ],"version":1}, 29 + sum(b_i) + (rows - 1) bytes. The cut is greedy: the first row of a
 * wave opens a part, and each next row joins the current part if the part stays <= L, else it opens a new part. So the parts
 * are unique, and no two consecutive parts of a wave could be merged within L. The parts are ordered by (wave, place in the
 * wave); document d is json[doc_off[d] .. doc_off[d+1]), back to back and not NUL-terminated. Every wave has at least one part,
 * and D <= the changed rows <= Q. With L >= the longest wave document, D = W, doc_wave[d] = d + 1, and json and doc_off are
 * byte for byte those of ka_plan_waves_json. json_cap = the bound of ka_plan_waves_json still suffices: every part holds at
 * least one row.
 * One document under a limit for a whole solve needs no other call: with max_broker_in >= the sum of the weights every changed
 * row is in wave 1, and wave 1 is cut into parts. Unchanged rows are in no part, which an operator does not submit anyway.
 * Checks, in this order: everything ka_plan_waves_json checks, in its order, with its codes and operands; then max_doc_bytes < 1,
 * or doc_wave or n_docs NULL with Q > 0: KA_ERR_BAD_ARG. On the device, after the plan's own row errors: a changed row whose
 * one-record document (29 + b_i bytes) exceeds L gives KA_ERR_LIMIT with a = the lowest such row (input order) and b = that
 * length clipped to INT_MAX; then a text longer than json_cap gives KA_ERR_LIMIT with a = min(json_cap, INT_MAX). On any error
 * *n_waves = *n_docs = 0 (when given) and nothing else is specified. W == 0 gives D = 0 and doc_off[0] = 0.
 * The Context's part caps (ka_ctx_set_part_caps) cut the parts finer: a row also opens a new part when the current one would
 * exceed Lr rows or, past its first row, Lx of data. The error checks and codes stay those above.
 * Synchronous; two synchronisations. The launches of ka_plan_waves_json, then, when W > 0, 4 more, and 2K - 1 more when the
 * widest wave has m >= 2 rows, K = the bit length of m - 1 (a pointer-doubling level per bit): they depend only on the bit
 * lengths of W and of m, and are the same with the part caps set or not. Follows the Context's wave rule
 * (ka_ctx_set_wave_rule); does not read or change the Context counters, parked counters, topic_base, the staged block, or the
 * last order / stage plans and timings. */
int32_t ka_plan_waves_json_parts(ka_ctx* ctx, int32_t T, const int64_t* part_off, const int32_t* part_id,
                                 const int64_t* rep_off, const int32_t* cur_broker, int32_t stride,
                                 const int32_t* new_len, const int32_t* new_broker, const int64_t* part_weight,
                                 int64_t max_broker_in, const char* names, const int64_t* name_off,
                                 char* json, int64_t json_cap, int64_t max_doc_bytes, int64_t* doc_off, int32_t* doc_wave,
                                 int32_t* n_docs, int32_t* wave, int32_t* n_waves, ka_wave_summary* summary,
                                 int32_t summary_cap, ka_status* st);

/* ka_plan_waves_json_parts under the rule of ka_plan_waves_send: the waves of ka_plan_waves_send_json, each cut into parts.
 *   T .. json_cap       exactly as ka_plan_waves_send_json takes them
 *   max_doc_bytes .. n_docs   exactly as ka_plan_waves_json_parts takes and writes them
 *   wave .. summary_cap   exactly as ka_plan_waves_send_json writes them
 * Checks: everything ka_plan_waves_send_json checks, in its order; then those ka_plan_waves_json_parts adds, in its order. The
 * launches of ka_plan_waves_send_json, and those ka_plan_waves_json_parts adds, with the part caps set or not. Follows the
 * Context's wave rule and its part caps (ka_ctx_set_part_caps), as ka_plan_waves_json_parts does. */
int32_t ka_plan_waves_send_json_parts(ka_ctx* ctx, int32_t T, const int64_t* part_off, const int32_t* part_id,
                                      const int64_t* rep_off, const int32_t* cur_broker, int32_t stride,
                                      const int32_t* new_len, const int32_t* new_broker, const int64_t* part_weight,
                                      int64_t max_broker_in, int32_t n_send, const int32_t* send_id, int64_t max_broker_out,
                                      const char* names, const int64_t* name_off, char* json, int64_t json_cap,
                                      int64_t max_doc_bytes, int64_t* doc_off, int32_t* doc_wave, int32_t* n_docs,
                                      int32_t* wave, int32_t* n_waves, ka_wave_summary* summary,
                                      ka_wave_send_summary* send_summary, int32_t summary_cap, ka_status* st);

/* ka_plan_waves_json_parts with every part's ROLLBACK document beside it: the document that puts exactly that part's partitions
 * back on their current lists, as kafka-reassign-partitions and the reference tool print them "in case a rollback is needed".
 * If part d stalls, rollback document d undoes it, however far the other parts have run: every changed row is in exactly one
 * part.
 *   T .. n_docs        exactly as ka_plan_waves_json_parts takes them
 *   back[back_cap]     host, required: the rollback text
 *   back_off[Q+1]      host, required when Q > 0; entries 0..D are written, back_off[0] = 0: rollback document d is
 *                      back[back_off[d] .. back_off[d+1]), back to back and not NUL-terminated
 *   wave .. summary_cap   exactly as ka_plan_waves_json_parts writes them
 * The rollback record of a changed row g is exactly the record the host's CURRENT ASSIGNMENT prints for that partition (Kafka
 * 0.10's ZkUtils.formatAsReassignmentJson key order): {"topic":"<name>","partition":<id>,"replicas":[<list>]}, the list being
 * cur_broker[rep_off[g] .. rep_off[g+1]) as given (duplicates, ids missing from the table and an empty list [] included); the
 * partition id and topic name as in the forward record. It is 39 + name + partition digits + list bytes, like the forward
 * record: the two differ only by the printed list. Rollback document d is {"version":1,"partitions":[ + the rollback records
 * of part d's rows, in part d's order, comma separated, + ]}: a 29-byte frame, like the forward one.
 * The paired cut: the greedy cut of ka_plan_waves_json_parts with one more condition, a row joins the current part only if BOTH
 * the part's document and its rollback document stay <= L. With S and R the exclusive prefixes of (record + comma) and
 * (rollback record + comma) over a wave's rows, rows i..j-1 make a part iff S[j] - S[i] <= L - 28 and R[j] - R[i] <= L - 28.
 * Both conditions are monotone in j, so the parts are unique and no two consecutive parts of a wave could be merged within L
 * on both sides. When no changed row's current list prints longer than its new list, the cut, json, doc_off and doc_wave are
 * exactly those of ka_plan_waves_json_parts; it differs where the rollback side is longer (a replication-factor reduction, a
 * move to shorter broker ids). With L >= the longest wave document on both sides, D = W and json is that of
 * ka_plan_waves_json. The plan, W, wave and the summaries are those of ka_plan_waves. The Context's part caps
 * (ka_ctx_set_part_caps) add their conditions to the paired cut; the rollback documents follow the parts.
 * Sufficient back_cap: the sum over rows of (79 + the name length of the row's topic), + 12 x rep_off[Q]. json_cap as before.
 * Checks, in this order: everything ka_plan_waves_json_parts checks, in its order; then back NULL, back_cap < 0, or back_off
 * NULL with Q > 0: KA_ERR_BAD_ARG. On the device: the plan's row errors; a changed row with 29 + max(record, rollback record)
 * > L: KA_ERR_LIMIT, a = the lowest such row (input order), b = that length clipped to INT_MAX; a text above json_cap:
 * KA_ERR_LIMIT, a = min(json_cap, INT_MAX); a rollback text above back_cap: KA_ERR_LIMIT, a = min(back_cap, INT_MAX). On any
 * error *n_waves = *n_docs = 0 (when given). W == 0 gives D = 0 and back_off[0] = 0.
 * Synchronous. The launches of ka_plan_waves_json_parts on the same inputs, and, when W > 0, 3 more (the rollback text's
 * length, scan and write passes; the part passes carry the rollback side without a launch of their own), with the part caps
 * set or not. Follows the
 * Context's wave rule (ka_ctx_set_wave_rule); does not read or change the Context counters, parked counters, topic_base, the staged block, or the last order / stage plans and timings. */
int32_t ka_plan_waves_json_parts_rollback(ka_ctx* ctx, int32_t T, const int64_t* part_off, const int32_t* part_id,
                                          const int64_t* rep_off, const int32_t* cur_broker, int32_t stride, const int32_t* new_len,
                                          const int32_t* new_broker, const int64_t* part_weight, int64_t max_broker_in,
                                          const char* names, const int64_t* name_off, char* json, int64_t json_cap,
                                          int64_t max_doc_bytes, int64_t* doc_off, int32_t* doc_wave, int32_t* n_docs, char* back,
                                          int64_t back_cap, int64_t* back_off, int32_t* wave, int32_t* n_waves,
                                          ka_wave_summary* summary, int32_t summary_cap, ka_status* st);

/* ka_plan_waves_json_parts_rollback under the rule of ka_plan_waves_send: ka_plan_waves_send_json_parts with the rollback
 * documents.
 *   T .. n_docs        exactly as ka_plan_waves_send_json_parts takes them
 *   back .. back_off   exactly as ka_plan_waves_json_parts_rollback takes and writes them
 *   wave .. summary_cap   exactly as ka_plan_waves_send_json_parts writes them
 * Checks: everything ka_plan_waves_send_json_parts checks, in its order; then those ka_plan_waves_json_parts_rollback adds, in
 * its order. The launches of ka_plan_waves_send_json_parts, and the 3 ka_plan_waves_json_parts_rollback adds, with the part
 * caps set or not. Follows the Context's wave rule and its part caps (ka_ctx_set_part_caps). */
int32_t ka_plan_waves_send_json_parts_rollback(ka_ctx* ctx, int32_t T, const int64_t* part_off, const int32_t* part_id,
                                               const int64_t* rep_off, const int32_t* cur_broker, int32_t stride,
                                               const int32_t* new_len, const int32_t* new_broker, const int64_t* part_weight,
                                               int64_t max_broker_in, int32_t n_send, const int32_t* send_id, int64_t max_broker_out,
                                               const char* names, const int64_t* name_off, char* json, int64_t json_cap,
                                               int64_t max_doc_bytes, int64_t* doc_off, int32_t* doc_wave, int32_t* n_docs,
                                               char* back, int64_t back_cap, int64_t* back_off, int32_t* wave, int32_t* n_waves,
                                               ka_wave_summary* summary, ka_wave_send_summary* send_summary, int32_t summary_cap,
                                               ka_status* st);

/* What one broker holds across a wave plan, in the weight's unit (ka_wave_broker_usage). Every field is int64, so the layout has
 * no padding. */
typedef struct ka_broker_usage {
    int64_t before;      /* before the plan starts: its base + the rows whose current list holds it */
    int64_t peak;        /* the most it holds at any wave 0..W ... */
    int64_t peak_wave;   /* ... and the lowest such wave (0 = before the plan starts) */
    int64_t after;       /* once every wave has run */
    int64_t over_wave;   /* the lowest wave in which it holds more than its capacity (0: already before), -1 when none */
} ka_broker_usage;

/* Every broker's disk usage across a wave plan: whether some broker runs out of disk PARTWAY through a plan, although it fits
 * both before and after. Kafka adds a new replica when a partition's reassignment starts and deletes the old one only when it
 * completes, so a broker that receives in one wave and drops in a later one holds both copies in between.
 *   Q .. part_weight   the rows exactly as ka_plan_waves takes them (1 <= stride <= 8; part_weight >= 0, or NULL = 1 per row)
 *   wave[Q]            host, required when Q > 0: every row's wave >= 0, e.g. the wave array of ka_plan_waves(_send), a plan the
 *                      caller reordered, or a whole solve as one document (changed ? 1 : 0). W = the largest entry (0 when Q == 0)
 *   n_use, use_id[n_use]   host; the USAGE TABLE, strictly ascending ids, 0 <= n_use <= 65535 (typically every broker of the
 *                      cluster before an exclusion: a drained broker holds data until its waves have run)
 *   use_base[n_use]    host, >= 0 per broker, or NULL = 0: what each broker holds beside the rows (e.g. topics outside the plan)
 *   use_cap[n_use]     host, >= 0 per broker, or NULL = no capacity
 *   usage[n_use]       host; usage[i] reports broker use_id[i]
 *   n_waves_out        host, required; *n_waves_out = W
 * The rule. Row g's RECEIVERS are the brokers of its new list that its current list lacks; its DROPPERS are the distinct
 * brokers of its current list that its new list lacks (a broker stores one copy: a duplicate id in a current list counts once).
 * For table broker b, with w_g the weight of row g:
 *   before[b]   = base[b] + sum of w_g over the rows whose current list holds b
 *   usage_b(v)  = before[b] + sum of w_g over the rows with 1 <= wave[g] <= v that b receives
 *                           - sum of w_g over the rows with 1 <= wave[g] < v that b drops,   v = 0 .. W
 * A receiver holds the new copy from the start of the row's wave, a dropper frees its copy only after that wave has ended: the
 * worst case inside a wave, so usage_b bounds what b holds under any order of the wave's parts. A row with wave 0 is not run:
 * it counts in before only. Then usage[i] = {before, peak = max_v usage(v), peak_wave = the lowest such v, after = usage(W) minus
 * the drops of wave W, over_wave = the lowest v with usage(v) > cap (-1 when none, or use_cap NULL)}. Ids outside the table are
 * not tracked.
 * Checks, in this order, before anything is enqueued: st NULL: KA_ERR_BAD_ARG (nothing written); ctx NULL: KA_ERR_NO_DEVICE;
 * Q < 0, stride < 1, n_use < 0, usage NULL with n_use > 0, n_waves_out NULL, rep_off not non-decreasing from 0, or a needed
 * array NULL: KA_ERR_BAD_ARG; stride > 8 (a = stride), Q >= 2^31 (a = INT_MAX) or n_use > 65535 (a = n_use): KA_ERR_LIMIT; use_id
 * not strictly ascending: KA_ERR_BAD_ARG; a negative weight, base or cap: KA_ERR_BAD_ARG; a new_len outside [0, stride] or a
 * negative wave: KA_ERR_BAD_ARG with a = the lowest such row; sum of the bases + sum over rows of w_g x (current + new list
 * lengths) > INT64_MAX, or Q x stride + rep_off[Q] > 2^31 - 1 (the replica events): KA_ERR_LIMIT. On the device, the lowest
 * failing row wins: a new list naming a broker twice, or a receiver of a row with wave[g] > 0 that the usage table lacks, gives
 * KA_ERR_BAD_ARG with a = the row and b = the broker id at the first such position of its list. On any error *n_waves_out = 0 and
 * usage is unspecified.
 * Synchronous; 2 kernel launches, and 3 per radix pass when W > 0: one per 8 bits of W + 1 and one per 8 bits of n_use - 1. Does
 * not read or change the Context counters, the broker table, parked counters, topic_base, the staged block, or the last order /
 * stage plans and timings. */
int32_t ka_wave_broker_usage(ka_ctx* ctx, int64_t Q, const int64_t* rep_off, const int32_t* cur_broker, int32_t stride,
                             const int32_t* new_len, const int32_t* new_broker, const int64_t* part_weight, const int32_t* wave,
                             int32_t n_use, const int32_t* use_id, const int64_t* use_base, const int64_t* use_cap,
                             ka_broker_usage* usage, int32_t* n_waves_out, ka_status* st);

/* The same solve split at the only point where topics stop being independent, for topic-sharded
 * multi-GPU runs (SURVEY.md §8e):
 *   ka_stage_dense_device  capacity, sticky fill, orphan spread (KAS:65-200) + per-broker histograms —
 *                          touches no Context state, so every GPU stages its own topic block concurrently;
 *   ka_order_device        leader-preference ordering (KAS:202-239) of the staged block against THIS ctx's
 *                          counters — a serial chain over all topics of the run, so rank g calls it after
 *                          importing the counters rank g-1 exported (ka_ctx_*_counters_device).
 * ka_solve_dense_device == stage + order. */
int32_t ka_stage_dense_device(ka_ctx* ctx, int32_t T, const int32_t* d_topic_hash, int32_t P, int32_t RF,
                              const int32_t* d_cur_broker, int32_t desired_rf, int32_t out_stride, void* stream);
int32_t ka_order_device(ka_ctx* ctx, int32_t* d_out_len, int32_t* d_out_broker, void* stream, ka_status* st);
/* Rows of <= 3 replicas are ordered by TWO independent chains: slot r reads and bumps only counter[.][r] (KAS:263-278 with
 * replicaId = r), slot 1 needs the slot-0 winners but slot 0 never waits for slot 1, and counter[.][2] is write-only
 * (a commutative sum added by the emit). A topic-sharded run therefore hands counter[.][0] to the next rank as soon as its
 * slot-0 chain is done, then counter[.][1]:
 *   ka_staged_slot_chains()   2 if the staged block is ordered by per-slot chains (all rows <= 3), else 0 (use ka_order_device)
 *   ka_order_slot_device()    the slot-0 (slot = 0) or slot-1 (slot = 1) chain of the staged block; slot 1 after slot 0
 *   ka_emit_device()          ordered records -> d_out_broker / d_out_len, adds counter[.][2]; ends the staged solve
 *                             (d_out_broker may be NULL only when the staged block has no rows; else KA_ERR_BAD_ARG)
 *   ka_ctx_{export,import}_counter_slot_device()  one counter column, d_column = N int32 on the device
 * ka_order_device == slot 0 (internal stream) overlapped with slot 1 + emit, sub-block by sub-block. */
int32_t ka_staged_slot_chains(ka_ctx* ctx);
int32_t ka_order_slot_device(ka_ctx* ctx, int32_t slot, void* stream);
int32_t ka_emit_device(ka_ctx* ctx, int32_t* d_out_len, int32_t* d_out_broker, void* stream, ka_status* st);
int32_t ka_ctx_export_counter_slot_device(ka_ctx* ctx, int32_t slot, int32_t* d_column, void* stream);
int32_t ka_ctx_import_counter_slot_device(ka_ctx* ctx, int32_t slot, const int32_t* d_column, void* stream);

/* Index of the staged block's first topic in the whole run: ka_status.topic_index of stage/order solves is reported
 * relative to the run (rank g of a topic-sharded job passes the number of topics owned by ranks < g), so that the ranks
 * can agree on the LOWEST failing topic of the run (KAG:173 aborts at the first throw). Default 0. */
int32_t ka_ctx_set_topic_base(ka_ctx* ctx, int32_t topic_base);

/* Synchronise the last asynchronous solve and return its status. */
int32_t ka_last_status(ka_ctx* ctx, ka_status* st);

/* ---- counters (Context.counter) -----------------------------------------------------------------
 * counter[i*slots + r] = Context.counter[broker_id[i]][r] for the CURRENT broker table (KAS:289-301:
 * absent == 0). slots = ka_ctx_counter_slots(). Used by tests and by the multi-GPU ring hand-off
 * (rank g imports what rank g-1 exported before ordering its own topics — S5 is a serial chain).
 * Values: any int32 may be set or imported. The rows and counters equal the reference's (whose counters are Java ints) as
 * long as every counter a run reads is below INT_MAX, e.g. every value at most INT_MAX minus the run's rows when it starts;
 * a bump past INT_MAX wraps, as the reference's does. Rows shorter than 3 are padded inside the chains with a dummy broker
 * whose counter is INT_MAX, listed after every real broker of the row and never bumped, so the dummy cannot win a slot
 * from a real broker at any counter value. */
int32_t ka_ctx_counter_slots(ka_ctx* ctx);
int32_t ka_ctx_get_counters(ka_ctx* ctx, int32_t* counter /* [N*slots] host */);
int32_t ka_ctx_set_counters(ka_ctx* ctx, const int32_t* counter /* [N*slots] host */);
/* device-to-device variants for NCCL plumbing: d_counter is a device buffer of N*slots int32. Stream contract: the copy
 * is enqueued on `stream`; pass the SAME stream as the stage/order calls (or order the streams yourself) — an import
 * must precede, and an export must follow, the ka_order_device it belongs to in stream order. */
int32_t ka_ctx_export_counters_device(ka_ctx* ctx, int32_t* d_counter, void* stream);
int32_t ka_ctx_import_counters_device(ka_ctx* ctx, const int32_t* d_counter, void* stream);

/* ---- instrumentation ----------------------------------------------------------------------------
 * Per-phase device times of the LAST solve, measured with CUDA events on the solve's stream.
 * ms[0]=sticky+spread kernel (S0-S4)  ms[1]=chunk tables of the level schedule (scan + fill; 0 when capacity is 1)
 * ms[2]=slot-0 leader-order chains (S5; first start .. last end)   ms[3]=H2D   ms[4]=D2H   ms[5]=total on stream
 * ms[6]=slot-1 chains + emits (first start .. last end; overlaps ms[2] in time)   ms[7]=wall time of all chains + emit
 * Enabled with ka_ctx_set_timing(ctx, 1); costs a few event records per solve. */
int32_t ka_ctx_set_timing(ka_ctx* ctx, int32_t enabled);
int32_t ka_ctx_last_timing(ka_ctx* ctx, float* ms /* [8] */);
/* Number of kernel launches issued by this ctx since creation (for bench.py's gpu_launches). */
int64_t ka_ctx_launch_count(ka_ctx* ctx);
/* The leader-order plan of the LAST solve call on this ctx (any entry point, including the staged and candidate calls):
 * plan[0] rec_kind (3 / 4 / 8)   plan[1] levels (0/1)   plan[2] chain threads   plan[3] ring_log2
 * plan[4] gctr (0/1)   plan[5] loop shape (0 general, 1 warp1, 2 single, 3 full)   plan[6] chain launches of the call
 * plan[7] candidates K (the clusters K of ka_solve_clusters; 0 for a single solve).
 * Cleared when a solve call passes its argument checks (ka_stage_dense_device starts a staged solve; its ka_order_device /
 * ka_order_slot_device calls add to it), so a call that launches no chain (a limit before any launch, or no rows) leaves
 * all zeros.
 * KA_ERR_BAD_ARG when ctx or plan is NULL. */
int32_t ka_ctx_last_order_plan(ka_ctx* ctx, int32_t* plan /* [8] */);
/* The sticky/spread plan (kernel A) of the LAST solve call on this ctx, from its last kernel A launch:
 * plan[0] load bytes per broker (1 / 2)   plan[1] levels (0/1)   plan[2] SM, the compile-time row bound (3 / 8)
 * plan[3] candidates K (0 for a single solve)   plan[4] warps per CTA   plan[5] grid.x (CTAs per candidate)
 * plan[6] bit mask of the id lookup modes of the call's broker tables (1: shared-memory LUT, 2: global LUT, 4: binary search)
 * plan[7] kernel A launches of the call.
 * Cleared as ka_ctx_last_order_plan is, so a call that launches no kernel A leaves all zeros. KA_ERR_BAD_ARG when ctx or
 * plan is NULL. */
int32_t ka_ctx_last_stage_plan(ka_ctx* ctx, int32_t* plan /* [8] */);

const char* ka_version(void);

#ifdef __cplusplus
}
#endif
#endif /* KASSIGN_H */
