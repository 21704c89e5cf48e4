// kassign_host.hpp — C++ host-side mirror of the reference's interface for the hot path, over the C ABI
// (include/kassign.h). Header-only; link with -lkassign.
//
//   kassign::KafkaTopicAssigner::generateAssignment   <->  siftscience.kafka.tools.KafkaTopicAssigner.generateAssignment
//                                                          (reference KafkaTopicAssigner.java:42-72)
//   kassign::solveTopics                              <->  the per-topic loop with ONE shared assigner
//                                                          (reference KafkaAssignmentGenerator.java:172-184)
//   kassign::solveTopicsJson                          <->  that loop + its org.json text, built on the device (KAG:172-186)
//   kassign::solveTopicsCandidates                    <->  that loop once per candidate broker set, each with a new
//                                                          assigner, in one device call (a decommission sweep)
//   kassign::scoreTopicsCandidates                    <->  the same sweep, reduced on the device to what each broker set
//                                                          would move and how evenly it spreads replicas and leaders
//   kassign::solveClusters                            <->  that loop once per cluster of a fleet, each with its own broker
//                                                          set and a new assigner, in one device call
//   kassign::solveClustersJson                        <->  the same fleet, with each cluster's org.json text built on the device
//   kassign::scoreClusters                            <->  the same fleet, reduced on the device to what each cluster would move
//                                                          and how evenly it spreads replicas and leaders
//   kassign::planWavesJson                            <->  planWaves with every wave's document built on the device
//   kassign::planWaveParts                            <->  planWavesJson with every wave cut into documents of at most a
//                                                          size limit (ZooKeeper's znode limit), cut on the device
//   kassign::planWavePartsRollback                    <->  planWaveParts with every part's rollback document (its partitions
//                                                          on their current lists), both sides under the limit
//   kassign::planWaves                                <->  a new assignment cut on the device into waves in which no broker
//                                                          receives more than a budget, one document per wave
//   kassign::setWaveRule                              <->  the wave rule of those plans: greedy, or first fit
//   kassign::setPartCaps                              <->  the most partitions and the most data one part of a wave holds
//   kassign::brokerUsage                              <->  what every broker holds across a wave plan: its peak, the wave of
//                                                          the peak and the first wave over its capacity
//   kassign::newAssignmentJson                        <->  the org.json emitter (KafkaAssignmentGenerator.java:169-186)
//
// Same argument meaning and error behaviour: failures are re-thrown as IllegalStateException /
// ArrayIndexOutOfBoundsException with the reference's message texts (KTA:58-60, 65-66, 67-69; KAS:183-184, 190-192).
// All compute runs in libkassign.so's CUDA kernels; there is no CPU fallback — without a GPU the constructor throws.
#pragma once
#include <algorithm>
#include <cstdint>
#include <map>
#include <memory>
#include <set>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../include/kassign.h"

namespace kassign {

struct IllegalStateException : std::logic_error { using std::logic_error::logic_error; };
struct ArrayIndexOutOfBoundsException : std::out_of_range { using std::out_of_range::out_of_range; };
struct KassignError : std::runtime_error {
    int code;
    KassignError(int c, const std::string& what) : std::runtime_error("kassign error " + std::to_string(c) + " " + what), code(c) {}
};

using Assignment = std::map<int, std::vector<int>>;  // partition -> replicas (leader first); TreeMap order

// Re-throw a ka_status as the reference's exception with the identical message.
inline void throwForStatus(const ka_status& st, const std::vector<std::string>& topicNames) {
    if (st.code == KA_OK) return;
    const std::string topic = (st.topic_index >= 0 && (size_t)st.topic_index < topicNames.size()) ? topicNames[st.topic_index] : "?";
    switch (st.code) {
    case KA_ERR_RF_MISMATCH:
        throw IllegalStateException("Topic " + topic + " has partition " + std::to_string(st.partition) +
                                    " with unexpected replication factor " + std::to_string(st.a));
    case KA_ERR_RF_NOT_POSITIVE:
        throw IllegalStateException("Topic " + topic + " does not have a positive replication factor!");
    case KA_ERR_RF_GT_BROKERS:
        throw IllegalStateException("Topic " + topic + " has a higher replication factor (" + std::to_string(st.a) +
                                    ") than available brokers!");
    case KA_ERR_UNASSIGNABLE:
        throw IllegalStateException("Partition " + std::to_string(st.partition) + " could not be fully assigned!");
    case KA_ERR_HASH_INDEX:
        throw ArrayIndexOutOfBoundsException(std::to_string(st.a));
    default:
        throw KassignError(st.code, "(topic_index=" + std::to_string(st.topic_index) + ")");
    }
}

// One topic of a run: name + current assignment.
struct TopicInput {
    std::string name;
    Assignment current;
};

struct TopicOutput {
    std::string name;
    Assignment assignment;
};

inline bool needsJsonEscape(const std::string& name);

class KafkaTopicAssigner {
public:
    // `new KafkaTopicAssigner()` (KTA:21-23): one Context per instance.
    explicit KafkaTopicAssigner(int device = 0) : ctx_(ka_ctx_create(device)), device_(device) {
        if (!ctx_) throw KassignError(KA_ERR_NO_DEVICE, "no usable CUDA device: kassign has no CPU fallback");
    }
    ~KafkaTopicAssigner() { ka_ctx_destroy(ctx_); }
    KafkaTopicAssigner(const KafkaTopicAssigner&) = delete;
    KafkaTopicAssigner& operator=(const KafkaTopicAssigner&) = delete;

    // generateAssignment(topic, currentAssignment, brokers, rackAssignment, desiredReplicationFactor) — KTA:42-44.
    Assignment generateAssignment(const std::string& topic, const Assignment& currentAssignment, const std::set<int>& brokers,
                                  const std::map<int, std::string>& rackAssignment, int desiredReplicationFactor) {
        std::vector<TopicInput> one{{topic, currentAssignment}};
        return solveTopics(one, brokers, rackAssignment, desiredReplicationFactor)[0].assignment;
    }

    // The KAG:172-184 loop as ONE batched device call: topics in order through this instance's Context.
    std::vector<TopicOutput> solveTopics(const std::vector<TopicInput>& topics, const std::set<int>& brokers,
                                         const std::map<int, std::string>& rackAssignment, int desiredReplicationFactor) {
        setBrokers(brokers, rackAssignment);
        const Flat f = flatten(topics, desiredReplicationFactor);
        ka_status st{};
        std::vector<TopicOutput> res = solveFlat(f, desiredReplicationFactor, st);
        throwForStatus(st, f.names);
        return res;
    }

    // One candidate broker set of a batched run: the `brokers` and `rackAssignment` of generateAssignment.
    struct Candidate {
        std::set<int> brokers;
        std::map<int, std::string> rackAssignment;
    };
    // What one candidate's run gave: its status (re-throw with throwForStatus) and, when that is KA_OK, the new assignment.
    struct CandidateResult {
        ka_status status;
        std::vector<TopicOutput> topics;
    };

    // The KAG:172-184 loop once per candidate broker set, each on a fresh Context (one new assigner per run), in ONE device
    // call (ka_solve_candidates): candidate k equals solveTopics(topics, brokers k, racks k) on a new KafkaTopicAssigner,
    // with the exception it would throw as its status. This instance's own Context is left alone. Rows of at most 3 replicas.
    std::vector<CandidateResult> solveTopicsCandidates(const std::vector<TopicInput>& topics, const std::vector<Candidate>& candidates,
                                                       int desiredReplicationFactor) {
        const Flat f = flatten(topics, desiredReplicationFactor);
        const int K = (int)candidates.size(), T = (int)topics.size();
        std::vector<int32_t> candOff{0}, ids, racks;
        for (const Candidate& c : candidates) addTable(c.brokers, c.rackAssignment, candOff, ids, racks);
        const size_t Q = f.partId.size();
        std::vector<int32_t> outLen((size_t)K * Q, 0), out((size_t)K * Q * f.stride, -1);
        std::vector<ka_status> st(std::max(K, 1));
        ka_solve_candidates(ctx_, K, candOff.data(), ids.data(), racks.data(), T, f.hash.data(), f.partOff.data(), f.partId.data(),
                            f.repOff.data(), f.cur.data(), desiredReplicationFactor, f.stride, outLen.data(), out.data(), st.data());
        return memberResults(st, K, f.stride, out, outLen, [&](int k) { return std::make_pair(&f, (int64_t)(k * Q)); });
    }

    // One cluster of a fleet: its topics and the arguments of its own run.
    struct ClusterInput {
        std::vector<TopicInput> topics;
        std::set<int> brokers;
        std::map<int, std::string> rackAssignment;
        int desiredReplicationFactor = -1;
    };

    // The KAG:172-184 loop once per cluster of a fleet, each with its own broker set on a fresh Context (one new assigner per
    // cluster), in ONE device call (ka_solve_clusters): cluster k equals solveTopics(its topics, brokers, racks, desired RF) on a
    // new KafkaTopicAssigner, with the exception it would throw as its status (topic_index counts from the cluster's first
    // topic). This instance's own Context is left alone. Rows of at most 3 replicas.
    std::vector<CandidateResult> solveClusters(const std::vector<ClusterInput>& clusters) {
        const int K = (int)clusters.size();
        const Fleet fl = flattenFleet(clusters);
        const int stride = fl.stride;
        const size_t Q = fl.partId.size();
        std::vector<int32_t> outLen(Q, 0), out(Q * stride, -1);
        std::vector<ka_status> st(std::max(K, 1));
        ka_solve_clusters(ctx_, K, fl.candOff.data(), fl.ids.data(), fl.racks.data(), fl.topicOff.data(), fl.desired.data(), fl.hash.data(),
                          fl.partOff.data(), fl.partId.data(), fl.repOff.data(), fl.cur.data(), stride, outLen.data(), out.data(), st.data());
        return memberResults(st, K, stride, out, outLen, [&](int k) { return std::make_pair(&fl.flat[k], fl.partOff[fl.topicOff[k]]); });
    }

    // What one cluster's JSON run gave: its status (re-throw with throwForStatus) and, when that is KA_OK, its "NEW ASSIGNMENT"
    // text.
    struct ClusterJson {
        ka_status status;
        std::string json;
    };

    // solveClusters with every cluster's text built on the device (ka_solve_clusters_json): cluster k equals solveTopicsJson(its
    // topics, brokers, racks, desired RF) on a new KafkaTopicAssigner, with the exception it would throw as its status. The
    // device call refuses clusters with a name ka_json_name_refused refuses or whose rows are wider than 3; those take
    // solveTopicsJson on a new assigner instead. This instance's own Context is left alone.
    std::vector<ClusterJson> solveClustersJson(const std::vector<ClusterInput>& clusters) {
        const int K = (int)clusters.size();
        const Fleet fl = flattenFleet(clusters);
        std::string names;
        std::vector<int64_t> nameOff(1, 0);
        int64_t cap = 0;
        for (const Flat& f : fl.flat) cap += appendNames(f, names, nameOff);
        std::unique_ptr<char[]> json(new char[std::max<int64_t>(cap, 1)]);
        std::vector<int64_t> jsonOff(K + 1, 0);
        std::vector<ka_status> st(std::max(K, 1));
        ka_solve_clusters_json(ctx_, K, fl.candOff.data(), fl.ids.data(), fl.racks.data(), fl.topicOff.data(), fl.desired.data(),
                               fl.hash.data(), fl.partOff.data(), fl.partId.data(), fl.repOff.data(), fl.cur.data(), names.data(),
                               nameOff.data(), json.get(), cap, jsonOff.data(), st.data());
        std::vector<ClusterJson> res(K);
        for (int k = 0; k < K; ++k) {
            bool escape = false;
            for (const auto& n : fl.flat[k].names) escape = escape || needsJsonEscape(n);
            if (escape || fl.flat[k].stride > 3) {
                KafkaTopicAssigner fresh(device_);
                res[k].json = fresh.solveTopicsJson(clusters[k].topics, clusters[k].brokers, clusters[k].rackAssignment,
                                                    clusters[k].desiredReplicationFactor, res[k].status);
                continue;
            }
            res[k].status = st[k];
            res[k].json.assign(json.get() + jsonOff[k], (size_t)(jsonOff[k + 1] - jsonOff[k]));
        }
        return res;
    }

    // What one candidate's run would move, and how it spreads the replicas (ka_move_summary); the per-broker maps are keyed by
    // broker id and hold every broker of the candidate (filled when asked for).
    struct CandidateScore {
        ka_status status;   // re-throw with throwForStatus; a failed candidate has a zero summary (max_broker_in_id = -1)
        ka_move_summary summary;
        std::map<int, int64_t> brokerReplicas, brokerLeaders, brokerIn;
    };

    // solveTopicsCandidates scored on the device (ka_score_candidates): per candidate the summary of what its new assignment
    // changes against `topics`' current one, instead of the assignment itself. weights: empty (1 per partition) or, per topic,
    // the weight of every partition (e.g. its size in bytes; a missing partition throws std::out_of_range).
    std::vector<CandidateScore> scoreTopicsCandidates(const std::vector<TopicInput>& topics, const std::vector<Candidate>& candidates,
                                                      int desiredReplicationFactor,
                                                      const std::vector<std::map<int, int64_t>>& weights = {}, bool perBroker = false) {
        const Flat f = flatten(topics, desiredReplicationFactor);
        const int K = (int)candidates.size(), T = (int)topics.size();
        std::vector<int32_t> candOff{0}, ids, racks;
        for (const Candidate& c : candidates) addTable(c.brokers, c.rackAssignment, candOff, ids, racks);
        std::vector<int64_t> w;
        if (!weights.empty()) {
            if (weights.size() != topics.size()) throw std::invalid_argument("one weight map per topic");
            for (int t = 0; t < T; ++t)
                for (const auto& e : topics[t].current) w.push_back(weights[t].at(e.first));
        }
        std::vector<ka_move_summary> summary(std::max(K, 1));
        std::vector<int64_t> brk[3];
        for (auto& a : brk) a.assign(perBroker ? ids.size() : 0, 0);
        std::vector<ka_status> st(std::max(K, 1));
        ka_score_candidates(ctx_, K, candOff.data(), ids.data(), racks.data(), T, f.hash.data(), f.partOff.data(), f.partId.data(),
                            f.repOff.data(), f.cur.data(), desiredReplicationFactor, f.stride, w.empty() ? nullptr : w.data(),
                            summary.data(), perBroker ? brk[0].data() : nullptr, perBroker ? brk[1].data() : nullptr,
                            perBroker ? brk[2].data() : nullptr, nullptr, nullptr, st.data());
        return memberScores(st, K, summary, perBroker ? brk : nullptr, candOff, ids);
    }

    // solveClusters scored on the device (ka_score_clusters): per cluster of the fleet the summary of what its new assignment
    // changes against its topics' current one, instead of the assignment itself. weights: empty (1 per partition) or, per
    // cluster, one map per topic with the weight of every partition, as scoreTopicsCandidates takes them.
    std::vector<CandidateScore> scoreClusters(const std::vector<ClusterInput>& clusters,
                                              const std::vector<std::vector<std::map<int, int64_t>>>& weights = {},
                                              bool perBroker = false) {
        const int K = (int)clusters.size();
        const Fleet fl = flattenFleet(clusters);
        std::vector<int64_t> w;
        if (!weights.empty()) {
            if (weights.size() != clusters.size()) throw std::invalid_argument("one list of weight maps per cluster");
            for (int k = 0; k < K; ++k) {
                if (weights[k].size() != clusters[k].topics.size()) throw std::invalid_argument("one weight map per topic");
                for (size_t t = 0; t < clusters[k].topics.size(); ++t)
                    for (const auto& e : clusters[k].topics[t].current) w.push_back(weights[k][t].at(e.first));
            }
        }
        std::vector<ka_move_summary> summary(std::max(K, 1));
        std::vector<int64_t> brk[3];
        for (auto& a : brk) a.assign(perBroker ? fl.ids.size() : 0, 0);
        std::vector<ka_status> st(std::max(K, 1));
        ka_score_clusters(ctx_, K, fl.candOff.data(), fl.ids.data(), fl.racks.data(), fl.topicOff.data(), fl.desired.data(), fl.hash.data(),
                          fl.partOff.data(), fl.partId.data(), fl.repOff.data(), fl.cur.data(), fl.stride, w.empty() ? nullptr : w.data(),
                          summary.data(), perBroker ? brk[0].data() : nullptr, perBroker ? brk[1].data() : nullptr,
                          perBroker ? brk[2].data() : nullptr, nullptr, nullptr, st.data());
        return memberScores(st, K, summary, perBroker ? brk : nullptr, fl.candOff, fl.ids);
    }

    // The wave rule of every planWaves* call of this instance (ka_ctx_set_wave_rule): KA_WAVE_GREEDY (the default: a broker's
    // waves only move forward) or KA_WAVE_FIRST_FIT (each partition in the earliest wave where its receivers and its leader still
    // have room, often fewer waves). Any other value throws KassignError(KA_ERR_BAD_ARG).
    void setWaveRule(int32_t rule) {
        const int32_t rc = ka_ctx_set_wave_rule(ctx_, rule);
        if (rc != KA_OK) throw KassignError(rc, "(wave rule " + std::to_string(rule) + ")");
    }
    int32_t waveRule() const { return ka_ctx_wave_rule(ctx_); }

    // The part caps of every planWaveParts / planWavePartsRollback call of this instance (ka_ctx_set_part_caps): a part holds at
    // most maxPartRows partitions, and moves at most maxPartIn (weight x the partition's new replicas, summed over the part)
    // unless it is a single partition; 0 is no cap. The plan and its summaries stay those of the uncapped call. A negative
    // value throws KassignError(KA_ERR_BAD_ARG) and leaves the caps as they were.
    void setPartCaps(int64_t maxPartRows, int64_t maxPartIn) {
        const int32_t rc = ka_ctx_set_part_caps(ctx_, maxPartRows, maxPartIn);
        if (rc != KA_OK)
            throw KassignError(rc, "(part caps " + std::to_string(maxPartRows) + ", " + std::to_string(maxPartIn) + ")");
    }
    // {maxPartRows, maxPartIn}, 0 where there is no cap.
    std::pair<int64_t, int64_t> partCaps() const {
        std::pair<int64_t, int64_t> caps{0, 0};
        ka_ctx_part_caps(ctx_, &caps.first, &caps.second);
        return caps;
    }

    // A new assignment cut into waves (ka_plan_waves): consecutive documents in which no broker of this instance's table receives
    // more than maxBrokerIn (weighted). waves[v] holds the changed partitions of wave v + 1, topics in input order, each
    // printable with newAssignmentJson; unchanged partitions are in no wave.
    struct WavePlan {
        ka_status status;   // re-throw with throwForStatus; on an error summary and waves are empty
        std::vector<ka_wave_summary> summary;
        std::vector<std::vector<TopicOutput>> waves;
        std::vector<ka_wave_send_summary> sendSummary;   // with a SendBudget: beside summary, one per wave
    };

    // A sender budget as well (ka_plan_waves_send): no partition leader (the first broker of its current list) sends more than
    // maxBrokerOut (weight x the partition's new replicas) per wave. sendBrokers, strictly ascending, must hold every such
    // leader: typically every broker of the cluster before an exclusion, since a drained broker still sends.
    struct SendBudget {
        int64_t maxBrokerOut;
        std::vector<int32_t> sendBrokers;
    };

    // `topics`' current assignment against `proposed` (the solveTopics output for them: the same topics and partitions, in the
    // same order), against the broker table of this instance's last solveTopics. weights: empty (1 per partition) or, per topic,
    // the weight of every partition, as scoreTopicsCandidates takes them.
    WavePlan planWaves(const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed, int64_t maxBrokerIn,
                       const std::vector<std::map<int, int64_t>>& weights = {}) {
        return planWavesWith(topics, proposed, maxBrokerIn, nullptr, weights);
    }
    // planWaves under a sender budget too; sendSummary is filled.
    WavePlan planWaves(const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed, int64_t maxBrokerIn,
                       const SendBudget& send, const std::vector<std::map<int, int64_t>>& weights = {}) {
        return planWavesWith(topics, proposed, maxBrokerIn, &send, weights);
    }

    // planWaves with every wave's document built on the device (ka_plan_waves_json): docs[v] equals
    // newAssignmentJson(planWaves(...).waves[v]). Topic names the device refuses (ka_json_name_refused) take the host emitter instead.
    struct WaveDocs {
        ka_status status;   // re-throw with throwForStatus; on an error summary and docs are empty
        std::vector<ka_wave_summary> summary;
        std::vector<std::string> docs;
        std::vector<ka_wave_send_summary> sendSummary;   // with a SendBudget: beside summary, one per wave
    };
    WaveDocs planWavesJson(const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed, int64_t maxBrokerIn,
                           const std::vector<std::map<int, int64_t>>& weights = {}) {
        return docsOf(waveDocuments(topics, proposed, maxBrokerIn, nullptr, false, nullptr, weights));
    }
    // planWavesJson under a sender budget too (ka_plan_waves_send_json); sendSummary is filled.
    WaveDocs planWavesJson(const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed, int64_t maxBrokerIn,
                           const SendBudget& send, const std::vector<std::map<int, int64_t>>& weights = {}) {
        return docsOf(waveDocuments(topics, proposed, maxBrokerIn, nullptr, false, &send, weights));
    }

    // planWavesJson with every wave cut into parts of at most maxDocBytes bytes (ka_plan_waves_json_parts): documents that run
    // one after the other, each small enough for the znode Kafka 0.10 writes it into (maxDocBytes = 1048575 under ZooKeeper's
    // default jute.maxbuffer). The cut is greedy: a wave's first partition opens a part, and each next partition of the wave
    // joins the current part while its document stays <= maxDocBytes, else it opens a new part. parts are in (wave, place in
    // the wave) order, partWave[d] the wave (1..W) of parts[d]; with maxDocBytes >= the longest wave document, parts equals
    // planWavesJson(...).docs. A partition whose one-record document exceeds maxDocBytes gives KA_ERR_LIMIT with a = its row
    // and b = that length. Topic names the device refuses (ka_json_name_refused) take the host emitter and the same cut on the host.
    // The part caps of setPartCaps cut finer on both paths: a partition also opens a new part when the current one holds
    // maxPartRows partitions, or would move more than maxPartIn.
    struct WaveParts {
        ka_status status;   // re-throw with throwForStatus; on an error summary, parts and partWave are empty
        std::vector<ka_wave_summary> summary;
        std::vector<std::string> parts;
        std::vector<int32_t> partWave;
        std::vector<ka_wave_send_summary> sendSummary;   // with a SendBudget: beside summary, one per wave
    };
    WaveParts planWaveParts(const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed, int64_t maxBrokerIn,
                            int64_t maxDocBytes, const std::vector<std::map<int, int64_t>>& weights = {}) {
        return partsOf(waveDocuments(topics, proposed, maxBrokerIn, &maxDocBytes, false, nullptr, weights));
    }
    // planWaveParts under a sender budget too (ka_plan_waves_send_json_parts); sendSummary is filled.
    WaveParts planWaveParts(const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed, int64_t maxBrokerIn,
                            int64_t maxDocBytes, const SendBudget& send, const std::vector<std::map<int, int64_t>>& weights = {}) {
        return partsOf(waveDocuments(topics, proposed, maxBrokerIn, &maxDocBytes, false, &send, weights));
    }

    // planWaveParts with every part's rollback document beside it (ka_plan_waves_json_parts_rollback): rollback[d] equals
    // kafkaReassignmentJson of parts[d]'s partitions, in parts[d]'s order, with their current lists, the document that undoes
    // part d whatever else has run. A partition joins a part only while both its document and its rollback document stay <=
    // maxDocBytes; when no current list prints longer than its new one, parts and partWave are those of planWaveParts. A
    // partition whose one-record document on either side exceeds maxDocBytes gives KA_ERR_LIMIT with a = its row and b = the
    // longer length. Topic names the device refuses (ka_json_name_refused) take the host emitters and the same cut on the host.
    // The part caps of setPartCaps apply as in planWaveParts.
    struct WaveRollback {
        ka_status status;   // re-throw with throwForStatus; on an error summary, parts, rollback and partWave are empty
        std::vector<ka_wave_summary> summary;
        std::vector<std::string> parts;
        std::vector<std::string> rollback;
        std::vector<int32_t> partWave;
        std::vector<ka_wave_send_summary> sendSummary;   // with a SendBudget: beside summary, one per wave
    };
    WaveRollback planWavePartsRollback(const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed,
                                       int64_t maxBrokerIn, int64_t maxDocBytes, const std::vector<std::map<int, int64_t>>& weights = {}) {
        return waveDocuments(topics, proposed, maxBrokerIn, &maxDocBytes, true, nullptr, weights);
    }
    // planWavePartsRollback under a sender budget too (ka_plan_waves_send_json_parts_rollback); sendSummary is filled.
    WaveRollback planWavePartsRollback(const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed,
                                       int64_t maxBrokerIn, int64_t maxDocBytes, const SendBudget& send,
                                       const std::vector<std::map<int, int64_t>>& weights = {}) {
        return waveDocuments(topics, proposed, maxBrokerIn, &maxDocBytes, true, &send, weights);
    }

    // What every broker of usageBrokers holds across a wave plan (ka_wave_broker_usage): its peak and the wave of the peak, and
    // the first wave in which it is over its capacity. `plan` is a planWaves result for these topics and proposed lists (or one
    // the caller built or reordered): each partition of plan.waves[v] runs in wave v + 1, every other partition is not run.
    // usageBrokers: strictly ascending (typically every broker of the cluster before an exclusion); base and capacity: empty (0 /
    // no capacity) or one entry per broker of usageBrokers; weights as planWaves takes them. usage is keyed by broker id and waves
    // = W; on an error usage is empty.
    struct BrokerUsage {
        ka_status status;   // re-throw with throwForStatus
        int32_t waves = 0;
        std::map<int32_t, ka_broker_usage> usage;
    };
    BrokerUsage brokerUsage(const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed, const WavePlan& plan,
                            const std::vector<int32_t>& usageBrokers, const std::vector<int64_t>& base = {},
                            const std::vector<int64_t>& capacity = {}, const std::vector<std::map<int, int64_t>>& weights = {}) {
        if ((!base.empty() && base.size() != usageBrokers.size()) || (!capacity.empty() && capacity.size() != usageBrokers.size()))
            throw std::invalid_argument("one base and one capacity per usage broker");
        const Flat f = flatten(topics, -1);
        const ProposedRows p = proposedRows(topics, proposed, weights);
        std::map<std::pair<std::string, int>, int32_t> waveOf;   // (topic, partition) -> its wave
        for (size_t v = 0; v < plan.waves.size(); ++v)
            for (const TopicOutput& t : plan.waves[v])
                for (const auto& e : t.assignment) waveOf[{t.name, e.first}] = (int32_t)v + 1;
        std::vector<int32_t> wave(f.partId.size(), 0);
        for (size_t t = 0; t < topics.size(); ++t)
            for (int64_t r = f.partOff[t]; r < f.partOff[t + 1]; ++r) {
                const auto it = waveOf.find({f.names[t], f.partId[r]});
                if (it != waveOf.end()) wave[r] = it->second;
            }
        BrokerUsage res{};
        std::vector<ka_broker_usage> usage(usageBrokers.size());
        ka_wave_broker_usage(ctx_, (int64_t)f.partId.size(), f.repOff.data(), f.cur.data(), p.stride, p.newLen.data(), p.newBroker.data(),
                             p.w.empty() ? nullptr : p.w.data(), wave.data(), (int32_t)usageBrokers.size(), usageBrokers.data(),
                             base.empty() ? nullptr : base.data(), capacity.empty() ? nullptr : capacity.data(), usage.data(), &res.waves,
                             &res.status);
        if (res.status.code != KA_OK) return res;
        for (size_t i = 0; i < usageBrokers.size(); ++i) res.usage[usageBrokers[i]] = usage[i];
        return res;
    }

private:
    // rowWave (when given) receives every row's wave, in the row order of flatten(topics).
    WavePlan planWavesWith(const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed, int64_t maxBrokerIn,
                           const SendBudget* send, const std::vector<std::map<int, int64_t>>& weights,
                           std::vector<int32_t>* rowWave = nullptr) {
        const Flat f = flatten(topics, -1);
        const ProposedRows p = proposedRows(topics, proposed, weights);
        const size_t Q = f.partId.size();
        WavePlan res{};
        std::vector<int32_t> wave(Q, 0);
        int32_t W = 0;
        // W never exceeds Q: min(Q, 64 k) summaries (40 bytes each) hold every plan in one call, but one of more than 64 k waves
        res.summary.resize(std::max<size_t>(1, std::min<size_t>(Q, 1 << 16)));
        auto plan = [&](int32_t* waveOut) {
            const int64_t* w = p.w.empty() ? nullptr : p.w.data();
            if (!send)
                return ka_plan_waves(ctx_, (int64_t)Q, f.repOff.data(), f.cur.data(), p.stride, p.newLen.data(), p.newBroker.data(), w,
                                     maxBrokerIn, waveOut, &W, res.summary.data(), (int32_t)res.summary.size(), &res.status);
            res.sendSummary.resize(res.summary.size());
            return ka_plan_waves_send(ctx_, (int64_t)Q, f.repOff.data(), f.cur.data(), p.stride, p.newLen.data(), p.newBroker.data(), w,
                                      maxBrokerIn, (int32_t)send->sendBrokers.size(), send->sendBrokers.data(), send->maxBrokerOut,
                                      waveOut, &W, res.summary.data(), res.sendSummary.data(), (int32_t)res.summary.size(),
                                      &res.status);
        };
        if (plan(wave.data()) == KA_OK && W > (int32_t)res.summary.size()) {
            res.summary.resize(W);
            plan(nullptr);
        }
        if (res.status.code != KA_OK) return WavePlan{res.status, {}, {}, {}};
        res.summary.resize(W);
        if (send) res.sendSummary.resize(W);
        if (rowWave) *rowWave = wave;
        res.waves.resize(W);
        std::vector<size_t> lastTopic(W, topics.size());   // the topic of each wave's last TopicOutput
        for (size_t t = 0; t < topics.size(); ++t)
            for (int64_t r = f.partOff[t]; r < f.partOff[t + 1]; ++r) {
                if (wave[r] == 0) continue;
                std::vector<TopicOutput>& doc = res.waves[wave[r] - 1];
                if (lastTopic[wave[r] - 1] != t) {
                    doc.push_back(TopicOutput{f.names[t], {}});
                    lastTopic[wave[r] - 1] = t;
                }
                doc.back().assignment[f.partId[r]] = std::vector<int>(p.newBroker.begin() + r * p.stride,
                                                                      p.newBroker.begin() + r * p.stride + p.newLen[r]);
            }
        return res;
    }
    // The one path of the six wave document entry points, each step once: with no maxDocBytes ka_plan_waves(_send)_json (parts
    // are the wave documents, partWave 1..W), else their _parts forms, and with rollback their _parts_rollback forms.
    WaveRollback waveDocuments(const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed, int64_t maxBrokerIn,
                               const int64_t* maxDocBytes, bool rollback, const SendBudget* send,
                               const std::vector<std::map<int, int64_t>>& weights);
    static WaveDocs docsOf(WaveRollback&& r) {
        return WaveDocs{r.status, std::move(r.summary), std::move(r.parts), std::move(r.sendSummary)};
    }
    static WaveParts partsOf(WaveRollback&& r) {
        return WaveParts{r.status, std::move(r.summary), std::move(r.parts), std::move(r.partWave), std::move(r.sendSummary)};
    }

public:

    // The KAG:172-186 loop and its "NEW ASSIGNMENT" text in one device call (ka_solve_json): only the text crosses PCIe.
    // Same solve and exceptions as solveTopics; the text equals newAssignmentJson(solveTopics(...)). Topic names the
    // device refuses (ka_json_name_refused) take that host emitter instead.
    std::string solveTopicsJson(const std::vector<TopicInput>& topics, const std::set<int>& brokers,
                                const std::map<int, std::string>& rackAssignment, int desiredReplicationFactor);
    // solveTopicsJson with the exception it would throw as `st` instead (the text is empty then).
    std::string solveTopicsJson(const std::vector<TopicInput>& topics, const std::set<int>& brokers,
                                const std::map<int, std::string>& rackAssignment, int desiredReplicationFactor, ka_status& st);

    ka_ctx* handle() { return ctx_; }

private:
    // The flat ragged layout of include/kassign.h (ka_solve / ka_solve_json inputs).
    struct Flat {
        std::vector<std::string> names;
        std::vector<int32_t> hash, partId, cur;
        std::vector<int64_t> partOff, repOff;
        int stride = 1;
    };
    // The proposed lists of a wave plan as ka_plan_waves takes them, in the row order of flatten(topics): newLen [Q], newBroker
    // [Q][stride] (stride = the longest proposed list, at least 1) and w [Q] (empty = 1 per row).
    struct ProposedRows {
        int stride = 1;
        std::vector<int32_t> newLen, newBroker;
        std::vector<int64_t> w;
    };
    // The name slab of f for the wave document calls (names, nameOff [T+1]); returns the json_cap kassign.h documents as
    // sufficient: per row 79 + 12·stride + its topic's name length.
    static int64_t waveNames(const Flat& f, int stride, std::string& names, std::vector<int64_t>& nameOff) {
        int64_t cap = 0;
        for (size_t t = 0; t < f.names.size(); ++t) {
            names += f.names[t];
            nameOff.push_back((int64_t)names.size());
            cap += (f.partOff[t + 1] - f.partOff[t]) * (79 + 12 * (int64_t)stride + (int64_t)f.names[t].size());
        }
        return cap;
    }
    static ProposedRows proposedRows(const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed,
                                     const std::vector<std::map<int, int64_t>>& weights) {
        if (proposed.size() != topics.size()) throw std::invalid_argument("one proposed topic per topic");
        if (!weights.empty() && weights.size() != topics.size()) throw std::invalid_argument("one weight map per topic");
        ProposedRows p;
        size_t Q = 0;
        for (size_t t = 0; t < topics.size(); ++t) {
            Q += topics[t].current.size();
            for (const auto& e : proposed[t].assignment) p.stride = std::max(p.stride, (int)e.second.size());
        }
        p.newLen.assign(Q, 0);
        p.newBroker.assign(Q * p.stride, -1);
        size_t g = 0;
        for (size_t t = 0; t < topics.size(); ++t)
            for (const auto& e : topics[t].current) {
                const std::vector<int>& l = proposed[t].assignment.at(e.first);
                p.newLen[g] = (int32_t)l.size();
                std::copy(l.begin(), l.end(), p.newBroker.begin() + g * p.stride);
                if (!weights.empty()) p.w.push_back(weights[t].at(e.first));
                ++g;
            }
        return p;
    }
    static Flat flatten(const std::vector<TopicInput>& topics, int desiredReplicationFactor) {
        const int T = (int)topics.size();
        Flat f;
        f.names.resize(T);
        f.hash.resize(T);
        f.partOff.assign(T + 1, 0);
        f.repOff.assign(1, 0);
        int maxLen = 0;
        for (int t = 0; t < T; ++t) {
            f.names[t] = topics[t].name;
            // the hash reads a C string: a NUL would leave it the hash of the name's prefix
            if (topics[t].name.find('\0') != std::string::npos)
                throw std::invalid_argument("topic " + std::to_string(t) + "'s name holds U+0000");
            f.hash[t] = ka_java_string_hash(topics[t].name.c_str());
            for (const auto& e : topics[t].current) {  // std::map: ascending partition == TreeMap order (KAS:107-110)
                f.partId.push_back(e.first);
                for (int b : e.second) f.cur.push_back(b);
                f.repOff.push_back((int64_t)f.cur.size());
                maxLen = std::max(maxLen, (int)e.second.size());
            }
            f.partOff[t + 1] = (int64_t)f.partId.size();
        }
        f.stride = std::max(1, std::max(maxLen, std::max(desiredReplicationFactor, 0)));
        return f;
    }
    // Rows of the flat layout (out[ΣP][stride], outLen[ΣP]) -> per-topic assignments.
    static std::vector<TopicOutput> unflatten(const Flat& f, int stride, const int32_t* out, const int32_t* outLen) {
        const int T = (int)f.names.size();
        std::vector<TopicOutput> res(T);
        for (int t = 0; t < T; ++t) {
            res[t].name = f.names[t];
            for (int64_t g = f.partOff[t]; g < f.partOff[t + 1]; ++g)
                res[t].assignment[f.partId[g]] = std::vector<int>(out + g * stride, out + g * stride + outLen[g]);
        }
        return res;
    }
    // ka_solve of `f` on this instance's Context into fresh rows -> per-topic assignments (none unless st is KA_OK).
    std::vector<TopicOutput> solveFlat(const Flat& f, int desiredReplicationFactor, ka_status& st) {
        const size_t Q = f.partId.size();
        std::vector<int32_t> outLen(Q, 0), out(Q * (size_t)f.stride, -1);
        ka_solve(ctx_, (int)f.names.size(), f.hash.data(), f.partOff.data(), f.partId.data(), f.repOff.data(), f.cur.data(),
                 desiredReplicationFactor, f.stride, outLen.data(), out.data(), &st);
        return st.code == KA_OK ? unflatten(f, f.stride, out.data(), outLen.data()) : std::vector<TopicOutput>();
    }
    // What each member of a batched call gave: its status and, when that is KA_OK, its rows. member(k) gives the member's flat
    // layout and its first row in out[.][stride] / outLen.
    template <class Member>
    static std::vector<CandidateResult> memberResults(const std::vector<ka_status>& st, int K, int stride, const std::vector<int32_t>& out,
                                                      const std::vector<int32_t>& outLen, Member member) {
        std::vector<CandidateResult> res(K);
        for (int k = 0; k < K; ++k) {
            res[k].status = st[k];
            if (st[k].code != KA_OK) continue;
            const std::pair<const Flat*, int64_t> m = member(k);
            res[k].topics = unflatten(*m.first, stride, out.data() + m.second * stride, outLen.data() + m.second);
        }
        return res;
    }
    // What each member of a scored call gave: its status, its summary and, when brk (the call's three per-broker arrays) is
    // given, its per-broker sums keyed by the ids of its table (ids[candOff[k] .. candOff[k + 1])).
    static std::vector<CandidateScore> memberScores(const std::vector<ka_status>& st, int K, const std::vector<ka_move_summary>& summary,
                                                    const std::vector<int64_t>* brk, const std::vector<int32_t>& candOff,
                                                    const std::vector<int32_t>& ids) {
        std::vector<CandidateScore> res(K);
        for (int k = 0; k < K; ++k) {
            res[k].status = st[k];
            res[k].summary = summary[k];
            if (brk)
                for (int i = candOff[k]; i < candOff[k + 1]; ++i) {
                    res[k].brokerReplicas[ids[i]] = brk[0][i];
                    res[k].brokerLeaders[ids[i]] = brk[1][i];
                    res[k].brokerIn[ids[i]] = brk[2][i];
                }
        }
        return res;
    }
    // Append the names of `f` to a name slab (names, nameOff) and return its document's sufficient size, documented in kassign.h:
    // 64 + per row (50 + 12·stride + its topic's name length).
    static int64_t appendNames(const Flat& f, std::string& names, std::vector<int64_t>& nameOff) {
        int64_t cap = 64;
        for (size_t t = 0; t < f.names.size(); ++t) {
            names += f.names[t];
            nameOff.push_back((int64_t)names.size());
            cap += (f.partOff[t + 1] - f.partOff[t]) * (50 + 12 * (int64_t)f.stride + (int64_t)f.names[t].size());
        }
        return cap;
    }
    // Rack index of every broker of `ids` (ascending) from the rack strings (ka_rack_indices, KAS:81-94).
    static int rackIndices(const std::vector<int32_t>& ids, const std::map<int, std::string>& racks, std::vector<int32_t>& rackIdx) {
        std::vector<const char*> names(ids.size(), nullptr);
        for (size_t i = 0; i < ids.size(); ++i) {
            auto it = racks.find(ids[i]);
            if (it != racks.end()) names[i] = it->second.c_str();
        }
        rackIdx.assign(ids.size(), 0);
        return ka_rack_indices((int32_t)ids.size(), ids.data(), names.data(), rackIdx.data());
    }
    // Append one broker set to the candidate tables of the C ABI (cand_off, broker_id, broker_rack); candOff starts as {0}.
    static void addTable(const std::set<int>& brokers, const std::map<int, std::string>& rackAssignment, std::vector<int32_t>& candOff,
                         std::vector<int32_t>& ids, std::vector<int32_t>& racks) {
        std::vector<int32_t> id(brokers.begin(), brokers.end()), rackIdx;
        const int rc = rackIndices(id, rackAssignment, rackIdx);
        if (rc != KA_OK) throw KassignError(rc, "ka_rack_indices");
        ids.insert(ids.end(), id.begin(), id.end());
        racks.insert(racks.end(), rackIdx.begin(), rackIdx.end());
        candOff.push_back((int32_t)ids.size());
    }
    void setBrokers(const std::set<int>& brokers, const std::map<int, std::string>& racks) {
        std::vector<int32_t> ids(brokers.begin(), brokers.end());  // std::set: ascending == TreeMap order (KAS:78)
        if (ids == ids_ && racks == racks_) return;
        std::vector<int32_t> rackIdx;
        int rc = rackIndices(ids, racks, rackIdx);
        if (rc == KA_OK) rc = ka_ctx_set_brokers(ctx_, (int32_t)ids.size(), ids.data(), rackIdx.data());
        if (rc != KA_OK) throw KassignError(rc, "ka_ctx_set_brokers");
        ids_ = ids;
        racks_ = racks;
    }
    // A fleet in the shared layout of ka_solve_clusters: every cluster's own flat layout, their broker tables, and the offsets
    // continued from one cluster to the next. stride = the largest cluster's.
    struct Fleet {
        std::vector<Flat> flat;
        std::vector<int32_t> candOff{0}, ids, racks, topicOff{0}, desired, hash, partId, cur;
        std::vector<int64_t> partOff{0}, repOff{0};
        int stride = 1;
    };
    static Fleet flattenFleet(const std::vector<ClusterInput>& clusters) {
        Fleet fl;
        for (const auto& cl : clusters) {
            fl.flat.push_back(flatten(cl.topics, cl.desiredReplicationFactor));
            const Flat& f = fl.flat.back();
            addTable(cl.brokers, cl.rackAssignment, fl.candOff, fl.ids, fl.racks);
            fl.desired.push_back(cl.desiredReplicationFactor);
            const int64_t row0 = fl.partOff.back(), rep0 = fl.repOff.back();
            fl.hash.insert(fl.hash.end(), f.hash.begin(), f.hash.end());
            for (size_t t = 1; t < f.partOff.size(); ++t) fl.partOff.push_back(row0 + f.partOff[t]);
            for (size_t g = 1; g < f.repOff.size(); ++g) fl.repOff.push_back(rep0 + f.repOff[g]);
            fl.partId.insert(fl.partId.end(), f.partId.begin(), f.partId.end());
            fl.cur.insert(fl.cur.end(), f.cur.begin(), f.cur.end());
            fl.topicOff.push_back((int32_t)fl.hash.size());
            fl.stride = std::max(fl.stride, f.stride);
        }
        return fl;
    }
    ka_ctx* ctx_;
    int device_;
    std::vector<int32_t> ids_;
    std::map<int, std::string> racks_;
};

// ---- JSON emission ------------------------------------------------------------------------------------------------
inline void appendInt(std::string& s, long long v) {
    char buf[24];
    int n = 0;
    unsigned long long u = v < 0 ? 0ULL - (unsigned long long)v : (unsigned long long)v;
    do { buf[n++] = (char)('0' + u % 10); u /= 10; } while (u);
    if (v < 0) s.push_back('-');
    while (n) s.push_back(buf[--n]);
}

// The quote of a UTF-8 string: escapes ", \, control chars and "</" (Kafka topic names never need it); with `wide`, also the
// chars org.json 20131018 JSONObject.quote() writes as \u plus four lowercase hex digits above ASCII: U+0080..U+009F and
// U+2000..U+20FF, whose UTF-8 forms ka_json_name_refused refuses. Every other byte is copied.
inline void appendQuotedAs(std::string& s, const std::string& v, bool wide) {
    static const char* hx = "0123456789abcdef";
    auto hex4 = [&](unsigned cp) { s += "\\u"; for (int k = 12; k >= 0; k -= 4) s.push_back(hx[(cp >> k) & 15]); };
    s.push_back('"');
    char prev = 0;
    for (size_t i = 0; i < v.size(); ++i) {
        const unsigned char c = (unsigned char)v[i];
        const unsigned char c1 = i + 1 < v.size() ? (unsigned char)v[i + 1] : 0, c2 = i + 2 < v.size() ? (unsigned char)v[i + 2] : 0;
        if (wide && c == 0xC2 && c1 >= 0x80 && c1 < 0xA0) {
            hex4(c1);
            ++i;
        } else if (wide && c == 0xE2 && c1 >= 0x80 && c1 < 0x84 && (c2 & 0xC0) == 0x80) {
            hex4(0x2000 | ((c1 & 0x3F) << 6) | (c2 & 0x3F));
            i += 2;
        } else {
            switch (c) {
            case '\\': case '"': s.push_back('\\'); s.push_back((char)c); break;
            case '/': if (prev == '<') s.push_back('\\'); s.push_back('/'); break;
            case '\b': s += "\\b"; break;
            case '\t': s += "\\t"; break;
            case '\n': s += "\\n"; break;
            case '\f': s += "\\f"; break;
            case '\r': s += "\\r"; break;
            default:
                if (c < 0x20) hex4(c);
                else s.push_back((char)c);
            }
        }
        prev = (char)c;
    }
    s.push_back('"');
}

// org.json JSONObject.quote(), for the records of KafkaAssignmentGenerator and the rack and host names of the broker list.
inline void appendQuoted(std::string& s, const std::string& v) { appendQuotedAs(s, v, true); }

// The quote of the CURRENT ASSIGNMENT and rollback records (Kafka's own encoder, not org.json): only the ASCII rewrites.
inline void appendKafkaQuoted(std::string& s, const std::string& v) { appendQuotedAs(s, v, false); }

// Key order of org.json 20131018 objects == java.util.HashMap iteration order of the keys (SURVEY §3.4; predicted for
// JDK >= 8, unverified without a JVM — isolated here so it can be corrected in one place):
//   top level: "partitions" (bucket 0) before "version" (13); per record: "partition" (3), "replicas" (6), "topic" (9).
inline void appendRecord(std::string& s, const std::string& topic, int partition, const int* replicas, size_t n) {
    s += "{\"partition\":";
    appendInt(s, partition);
    s += ",\"replicas\":[";
    for (size_t i = 0; i < n; ++i) {
        if (i) s.push_back(',');
        appendInt(s, replicas[i]);
    }
    s += "],\"topic\":";
    appendQuoted(s, topic);
    s.push_back('}');
}

// A partition's record in Kafka 0.10 ZkUtils.formatAsReassignmentJson order (the "CURRENT ASSIGNMENT" and rollback records):
// scala Map literals keep insertion order for <= 4 entries: topic, partition, replicas.
inline void appendCurrentRecord(std::string& s, const std::string& topic, int partition, const int* replicas, size_t n) {
    s += "{\"topic\":";
    appendKafkaQuoted(s, topic);
    s += ",\"partition\":";
    appendInt(s, partition);
    s += ",\"replicas\":[";
    for (size_t i = 0; i < n; ++i) {
        if (i) s.push_back(',');
        appendInt(s, replicas[i]);
    }
    s += "]}";
}

inline std::string newAssignmentJson(const std::vector<TopicOutput>& topics) {
    std::string s = "{\"partitions\":[";
    bool first = true;
    for (const auto& t : topics)
        for (const auto& e : t.assignment) {  // ascending partition, topics in loop order (KAG:173-183)
            if (!first) s.push_back(',');
            first = false;
            appendRecord(s, t.name, e.first, e.second.data(), e.second.size());
        }
    s += "],\"version\":1}";  // KAFKA_FORMAT_VERSION (KAG:49)
    return s;
}

// A name the device emitters refuse (ka_json_name_refused: a character org.json's JSONObject.quote() may rewrite, or '/'):
// such names take the host emitter, appendQuoted.
inline bool needsJsonEscape(const std::string& name) { return ka_json_name_refused(name.data(), (int64_t)name.size()) >= 0; }

inline std::string KafkaTopicAssigner::solveTopicsJson(const std::vector<TopicInput>& topics, const std::set<int>& brokers,
                                                       const std::map<int, std::string>& rackAssignment,
                                                       int desiredReplicationFactor) {
    ka_status st{};
    std::string json = solveTopicsJson(topics, brokers, rackAssignment, desiredReplicationFactor, st);
    std::vector<std::string> names;
    for (const auto& t : topics) names.push_back(t.name);
    throwForStatus(st, names);
    return json;
}

inline std::string KafkaTopicAssigner::solveTopicsJson(const std::vector<TopicInput>& topics, const std::set<int>& brokers,
                                                       const std::map<int, std::string>& rackAssignment, int desiredReplicationFactor,
                                                       ka_status& st) {
    setBrokers(brokers, rackAssignment);
    const Flat f = flatten(topics, desiredReplicationFactor);
    const int T = (int)topics.size();
    st = ka_status{};
    for (const auto& t : topics)
        if (needsJsonEscape(t.name)) {   // the host emitter over the rows of solveTopics
            const std::vector<TopicOutput> rows = solveFlat(f, desiredReplicationFactor, st);
            return st.code == KA_OK ? newAssignmentJson(rows) : std::string();
        }
    std::string names;
    std::vector<int64_t> nameOff(1, 0);
    const int64_t cap = appendNames(f, names, nameOff);
    std::unique_ptr<char[]> json(new char[cap]);
    int64_t bytes = 0;
    ka_solve_json(ctx_, T, f.hash.data(), f.partOff.data(), f.partId.data(), f.repOff.data(), f.cur.data(), desiredReplicationFactor,
                  names.data(), nameOff.data(), json.get(), cap, &bytes, &st);
    return std::string(json.get(), (size_t)bytes);
}

// Kafka 0.10 ZkUtils.formatAsReassignmentJson shape (used for "CURRENT ASSIGNMENT:", KAG:103-111): scala Map literals keep
// insertion order for <= 4 entries: version, partitions / topic, partition, replicas.
inline std::string kafkaReassignmentJson(const std::vector<TopicInput>& topics) {
    std::string s = "{\"version\":1,\"partitions\":[";
    bool first = true;
    for (const auto& t : topics)
        for (const auto& e : t.current) {
            if (!first) s.push_back(',');
            first = false;
            appendCurrentRecord(s, t.name, e.first, e.second.data(), e.second.size());
        }
    s += "]}";
    return s;
}

inline KafkaTopicAssigner::WaveRollback KafkaTopicAssigner::waveDocuments(const std::vector<TopicInput>& topics,
                                                                          const std::vector<TopicOutput>& proposed, int64_t maxBrokerIn,
                                                                          const int64_t* maxDocBytes, bool rollback,
                                                                          const SendBudget* send,
                                                                          const std::vector<std::map<int, int64_t>>& weights) {
    const Flat f = flatten(topics, -1);
    const ProposedRows p = proposedRows(topics, proposed, weights);
    const size_t Q = f.partId.size();
    WaveRollback res{};
    if (std::any_of(topics.begin(), topics.end(), [](const TopicInput& t) { return needsJsonEscape(t.name); })) {
        // the host emitters over the rows of planWaves, cut by the same greedy rule; no limit: every wave one part
        std::vector<int32_t> rowWave;
        const WavePlan plan = planWavesWith(topics, proposed, maxBrokerIn, send, weights, &rowWave);
        const int64_t L = maxDocBytes ? *maxDocBytes : INT64_MAX;
        res = WaveRollback{plan.status, plan.summary, {}, {}, {}, plan.sendSummary};
        if (res.status.code == KA_OK && L < 1) res.status.code = KA_ERR_BAD_ARG;
        if (res.status.code != KA_OK) return WaveRollback{res.status, {}, {}, {}, {}, {}};
        // the part caps of ka_ctx_set_part_caps: the most records of a part, the most data it moves (past its first record)
        const std::pair<int64_t, int64_t> caps = maxDocBytes ? partCaps() : std::pair<int64_t, int64_t>{0, 0};
        const int64_t maxRows = caps.first > 0 ? caps.first : INT64_MAX, maxIn = caps.second > 0 ? caps.second : INT64_MAX;
        std::vector<std::vector<std::pair<std::string, std::string>>> recs(plan.summary.size());   // (record, rollback record)
        std::vector<std::vector<int64_t>> moved(plan.summary.size());   // every record's weight x its receivers
        for (size_t t = 0; t < f.names.size(); ++t)
            for (int64_t r = f.partOff[t]; r < f.partOff[t + 1]; ++r) {
                if (rowWave[r] == 0) continue;
                int64_t receivers = 0;
                for (int32_t j = 0; j < p.newLen[r]; ++j)
                    receivers += std::find(f.cur.begin() + f.repOff[r], f.cur.begin() + f.repOff[r + 1], p.newBroker[r * p.stride + j]) ==
                                 f.cur.begin() + f.repOff[r + 1];
                moved[rowWave[r] - 1].push_back(receivers * (p.w.empty() ? 1 : p.w[r]));
                std::string rec, back;
                appendRecord(rec, f.names[t], f.partId[r], p.newBroker.data() + r * p.stride, (size_t)p.newLen[r]);
                if (rollback)
                    appendCurrentRecord(back, f.names[t], f.partId[r], f.cur.data() + f.repOff[r], (size_t)(f.repOff[r + 1] - f.repOff[r]));
                const int64_t longest = 29 + (int64_t)std::max(rec.size(), back.size());
                if (longest > L) {
                    ka_status st{};
                    st.code = KA_ERR_LIMIT;
                    st.a = (int32_t)r;
                    st.b = (int32_t)std::min<int64_t>(longest, INT32_MAX);
                    return WaveRollback{st, {}, {}, {}, {}, {}};
                }
                recs[rowWave[r] - 1].emplace_back(std::move(rec), std::move(back));
            }
        for (size_t v = 0; v < recs.size(); ++v) {
            // the current part's two document sizes, 0 before the wave's first; without rollback the empty back side never binds;
            // its records and the data they move
            int64_t size = 0, backSize = 0, rows = 0, in = 0;
            for (size_t k = 0; k < recs[v].size(); ++k) {
                const auto& rb = recs[v][k];
                const int64_t n = (int64_t)rb.first.size(), m = (int64_t)rb.second.size(), a = moved[v][k];
                if (size > 0 && size + 1 + n <= L && backSize + 1 + m <= L && rows < maxRows && in + a <= maxIn) {
                    res.parts.back().insert(res.parts.back().size() - 14, "," + rb.first);
                    if (rollback) res.rollback.back().insert(res.rollback.back().size() - 2, "," + rb.second);
                    size += 1 + n;
                    backSize += 1 + m;
                    rows += 1;
                    in += a;
                } else {
                    res.parts.push_back("{\"partitions\":[" + rb.first + "],\"version\":1}");
                    if (rollback) res.rollback.push_back("{\"version\":1,\"partitions\":[" + rb.second + "]}");
                    res.partWave.push_back((int32_t)v + 1);
                    size = 29 + n;
                    backSize = 29 + m;
                    rows = 1;
                    in = a;
                }
            }
        }
        return res;
    }
    std::string names;
    std::vector<int64_t> nameOff(1, 0);
    const int64_t cap = waveNames(f, p.stride, names, nameOff);
    int64_t backCap = 0;
    if (rollback) {   // per row 79 + its topic's name, 12 per current broker
        backCap = 12 * (int64_t)f.cur.size();
        for (size_t t = 0; t < f.names.size(); ++t) backCap += (f.partOff[t + 1] - f.partOff[t]) * (79 + (int64_t)f.names[t].size());
    }
    std::unique_ptr<char[]> json(new char[std::max<int64_t>(cap, 1)]), back(rollback ? new char[std::max<int64_t>(backCap, 1)] : nullptr);
    std::vector<int64_t> docOff(Q + 1, 0), backOff(Q + 1, 0);
    std::vector<int32_t> docWave(std::max<size_t>(Q, 1), 0);
    res.summary.resize(std::max<size_t>(Q, 1));   // W never exceeds Q: one call
    if (send) res.sendSummary.resize(res.summary.size());
    int32_t W = 0, D = 0;
    const int32_t T = (int32_t)topics.size(), S = (int32_t)res.summary.size();
    const int64_t *po = f.partOff.data(), *ro = f.repOff.data(), *w = p.w.empty() ? nullptr : p.w.data();
    const int32_t *pid = f.partId.data(), *cu = f.cur.data(), *nl = p.newLen.data(), *nb = p.newBroker.data();
    const int32_t nSend = send ? (int32_t)send->sendBrokers.size() : 0;
    const int32_t* sendId = send ? send->sendBrokers.data() : nullptr;
    const int64_t C = send ? send->maxBrokerOut : 0;
    ka_wave_summary* sum = res.summary.data();
    ka_wave_send_summary* sendSum = res.sendSummary.data();
    if (!maxDocBytes && !send)
        ka_plan_waves_json(ctx_, T, po, pid, ro, cu, p.stride, nl, nb, w, maxBrokerIn, names.data(), nameOff.data(), json.get(), cap,
                           docOff.data(), nullptr, &W, sum, S, &res.status);
    else if (!maxDocBytes)
        ka_plan_waves_send_json(ctx_, T, po, pid, ro, cu, p.stride, nl, nb, w, maxBrokerIn, nSend, sendId, C, names.data(), nameOff.data(),
                                json.get(), cap, docOff.data(), nullptr, &W, sum, sendSum, S, &res.status);
    else if (!rollback && !send)
        ka_plan_waves_json_parts(ctx_, T, po, pid, ro, cu, p.stride, nl, nb, w, maxBrokerIn, names.data(), nameOff.data(), json.get(), cap,
                                 *maxDocBytes, docOff.data(), docWave.data(), &D, nullptr, &W, sum, S, &res.status);
    else if (!rollback)
        ka_plan_waves_send_json_parts(ctx_, T, po, pid, ro, cu, p.stride, nl, nb, w, maxBrokerIn, nSend, sendId, C, names.data(),
                                      nameOff.data(), json.get(), cap, *maxDocBytes, docOff.data(), docWave.data(), &D, nullptr, &W, sum,
                                      sendSum, S, &res.status);
    else if (!send)
        ka_plan_waves_json_parts_rollback(ctx_, T, po, pid, ro, cu, p.stride, nl, nb, w, maxBrokerIn, names.data(), nameOff.data(),
                                          json.get(), cap, *maxDocBytes, docOff.data(), docWave.data(), &D, back.get(), backCap,
                                          backOff.data(), nullptr, &W, sum, S, &res.status);
    else
        ka_plan_waves_send_json_parts_rollback(ctx_, T, po, pid, ro, cu, p.stride, nl, nb, w, maxBrokerIn, nSend, sendId, C, names.data(),
                                               nameOff.data(), json.get(), cap, *maxDocBytes, docOff.data(), docWave.data(), &D,
                                               back.get(), backCap, backOff.data(), nullptr, &W, sum, sendSum, S, &res.status);
    if (res.status.code != KA_OK) return WaveRollback{res.status, {}, {}, {}, {}, {}};
    if (!maxDocBytes) {   // one document per wave
        D = W;
        for (int32_t v = 0; v < W; ++v) docWave[v] = v + 1;
    }
    res.summary.resize(W);
    if (send) res.sendSummary.resize(W);
    for (int32_t d = 0; d < D; ++d) {
        res.parts.emplace_back(json.get() + docOff[d], (size_t)(docOff[d + 1] - docOff[d]));
        if (rollback) res.rollback.emplace_back(back.get() + backOff[d], (size_t)(backOff[d + 1] - backOff[d]));
    }
    res.partWave.assign(docWave.begin(), docWave.begin() + D);
    return res;
}

}  // namespace kassign
