// test_cluster_scores.cpp — KafkaTopicAssigner::scoreClusters against the per-cluster scores it replaces: every cluster equals
// scoreTopicsCandidates on a new KafkaTopicAssigner with that cluster's one broker set (summary, per-broker sums and status),
// with and without weights; failing clusters are zero and carry their exception. Needs a GPU (kassign has no CPU fallback).
// Exit code 0 = all passed.
#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include "kassign_host.hpp"

using kassign::KafkaTopicAssigner;
using kassign::TopicInput;
using Cluster = KafkaTopicAssigner::ClusterInput;
using Weights = std::vector<std::map<int, int64_t>>;

static int failures = 0;
#define CHECK(cond)                                                              \
    do {                                                                         \
        if (!(cond)) { std::fprintf(stderr, "FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); ++failures; } \
    } while (0)

// A seeded ragged run: 1..maxP partitions per topic with sparse ids, replication factor 1..3, lists on brokers 1..nb.
static std::vector<TopicInput> makeTopics(unsigned seed, int T, int nb, int maxP) {
    auto next = [&]() { seed = seed * 1103515245u + 12345u; return (int)((seed >> 8) & 0xFFFF); };
    std::vector<TopicInput> topics(T);
    for (int t = 0; t < T; ++t) {
        topics[t].name = "svc.topic-" + std::to_string(t);
        const int P = 1 + next() % maxP, rf = 1 + next() % 3;
        int id = next() % 5;
        for (int p = 0; p < P; ++p, id += 1 + next() % 3) {
            std::vector<int> lst;
            while ((int)lst.size() < rf) {
                const int b = 1 + next() % nb;
                if (std::find(lst.begin(), lst.end(), b) == lst.end()) lst.push_back(b);
            }
            topics[t].current[id] = lst;
        }
    }
    return topics;
}

static Cluster cluster(std::vector<TopicInput> topics, int lo, int hi, int racks, int desired = -1) {
    Cluster c;
    c.topics = std::move(topics);
    for (int b = lo; b <= hi; ++b) {
        c.brokers.insert(b);
        if (racks > 0) c.rackAssignment[b] = "rack" + std::to_string(b % racks);
    }
    c.desiredReplicationFactor = desired;
    return c;
}

static Weights weightsOf(const std::vector<TopicInput>& topics, unsigned seed) {
    Weights w(topics.size());
    for (size_t t = 0; t < topics.size(); ++t)
        for (const auto& p : topics[t].current) { seed = seed * 1103515245u + 12345u; w[t][p.first] = (int64_t)(seed >> 4) << 12; }
    return w;
}

static bool sameSummary(const ka_move_summary& a, const ka_move_summary& b) {
    return a.rows_changed == b.rows_changed && a.rows_moved == b.rows_moved && a.leaders_changed == b.leaders_changed &&
           a.replicas_added == b.replicas_added && a.replicas_dropped == b.replicas_dropped && a.max_broker_in == b.max_broker_in &&
           a.max_broker_in_id == b.max_broker_in_id && a.max_broker_replicas == b.max_broker_replicas &&
           a.min_broker_replicas == b.min_broker_replicas && a.max_broker_leaders == b.max_broker_leaders &&
           a.min_broker_leaders == b.min_broker_leaders;
}

static bool sameStatus(const ka_status& a, const ka_status& b) {
    return a.code == b.code && a.topic_index == b.topic_index && a.partition == b.partition && a.a == b.a && a.b == b.b;
}

static void testClustersEqualOneTableEach() {
    const std::vector<Cluster> fleet = {
        cluster(makeTopics(7u, 60, 30, 12), 1, 30, 0),          // no racks
        cluster(makeTopics(8u, 20, 24, 40), 1, 24, 4, 2),       // four racks, RF 2
        cluster(makeTopics(9u, 0, 10, 8), 1, 10, 0),            // no topics
        cluster(makeTopics(10u, 40, 40, 12), 3, 40, 5),         // expansion
        cluster(makeTopics(11u, 30, 30, 12), 1, 2, 0),          // fewer brokers than RF 3: "higher replication factor"
        cluster(makeTopics(12u, 30, 30, 12), 1, 30, 2),         // RF 3 over two racks: "could not be fully assigned"
        cluster(makeTopics(13u, 10, 30, 12), 1, 0, 0),          // no broker at all
        cluster(makeTopics(14u, 50, 30, 12), 5, 30, 3, 1),      // shrinks to RF 1
    };
    std::vector<Weights> weights;
    for (size_t k = 0; k < fleet.size(); ++k) weights.push_back(weightsOf(fleet[k].topics, 5u + (unsigned)k));
    KafkaTopicAssigner mine;
    for (bool weighted : {true, false}) {
        const auto res = mine.scoreClusters(fleet, weighted ? weights : std::vector<Weights>(), true);
        CHECK(res.size() == fleet.size());
        int solved = 0, changed = 0;
        for (size_t k = 0; k < fleet.size() && k < res.size(); ++k) {
            KafkaTopicAssigner fresh;
            const KafkaTopicAssigner::Candidate one{fleet[k].brokers, fleet[k].rackAssignment};
            const auto e = fresh.scoreTopicsCandidates(fleet[k].topics, {one}, fleet[k].desiredReplicationFactor,
                                                       weighted ? weights[k] : Weights(), true)[0];
            CHECK(sameStatus(res[k].status, e.status));
            if (!sameSummary(res[k].summary, e.summary)) {
                std::fprintf(stderr, "cluster %zu (weighted %d): summaries differ\n", k, (int)weighted);
                ++failures;
            }
            CHECK(res[k].brokerReplicas == e.brokerReplicas && res[k].brokerLeaders == e.brokerLeaders && res[k].brokerIn == e.brokerIn);
            if (res[k].status.code != KA_OK) {
                for (const auto& b : res[k].brokerReplicas) CHECK(b.second == 0);
                CHECK(res[k].summary.max_broker_in_id == -1 && res[k].summary.rows_changed == 0);
            } else {
                ++solved;
                changed += res[k].summary.rows_changed > 0;
            }
        }
        CHECK(solved >= 4);
        CHECK(changed >= 2);
        CHECK(res[2].status.code == KA_OK && res[2].summary.max_broker_in_id == -1 && res[2].summary.rows_changed == 0 &&
              res[2].summary.max_broker_replicas == 0);   // no topics: solved, with the empty summary
    }
    // a failing cluster re-throws its exception
    std::vector<std::string> names;
    for (const auto& t : fleet[4].topics) names.push_back(t.name);
    const auto res = mine.scoreClusters({fleet[4]});
    try { kassign::throwForStatus(res[0].status, names); CHECK(false); }
    catch (const kassign::IllegalStateException& e) { CHECK(std::string(e.what()).find("higher replication factor") != std::string::npos); }
}

int main() {
    try {
        testClustersEqualOneTableEach();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 2;
    }
    std::printf("%s (%d failure%s)\n", failures ? "FAILED" : "OK", failures, failures == 1 ? "" : "s");
    return failures ? 1 : 0;
}
