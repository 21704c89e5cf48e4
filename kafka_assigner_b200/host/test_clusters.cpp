// test_clusters.cpp — KafkaTopicAssigner::solveClusters against the per-cluster runs it replaces: every cluster equals
// solveTopics on a new KafkaTopicAssigner with its own broker set and desired replication factor, a failing cluster re-throws
// the reference's message text (KTA:58-60, 65-66, 67-69; KAS:183-184, 190-192) without touching the others, and the
// instance's own Context is left alone. Needs a GPU (kassign has no CPU fallback). Exit code 0 = all passed.
#include <cstdio>
#include <cstdlib>

#include "kassign_host.hpp"

using kassign::KafkaTopicAssigner;
using kassign::TopicInput;
using kassign::TopicOutput;
using Cluster = KafkaTopicAssigner::ClusterInput;

static int failures = 0;
#define CHECK(cond)                                                              \
    do {                                                                         \
        if (!(cond)) { std::fprintf(stderr, "FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); ++failures; } \
    } while (0)

static bool sameTopics(const std::vector<TopicOutput>& a, const std::vector<TopicOutput>& b) {
    if (a.size() != b.size()) return false;
    for (size_t t = 0; t < a.size(); ++t)
        if (a[t].name != b[t].name || a[t].assignment != b[t].assignment) return false;
    return true;
}

// A seeded ragged run: 1..40 partitions per topic with sparse ids, replication factor 1..3, lists on brokers 1..nb.
static std::vector<TopicInput> makeTopics(unsigned seed, int T, int nb) {
    auto next = [&]() { seed = seed * 1103515245u + 12345u; return (int)((seed >> 8) & 0xFFFF); };
    std::vector<TopicInput> topics(T);
    for (int t = 0; t < T; ++t) {
        topics[t].name = "svc.topic-" + std::to_string(t);
        const int P = 1 + next() % 40, rf = 1 + next() % 3;
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

static std::string messageOf(const ka_status& st, const std::vector<TopicInput>& topics) {
    std::vector<std::string> names;
    for (const auto& t : topics) names.push_back(t.name);
    try { kassign::throwForStatus(st, names); } catch (const std::exception& e) { return e.what(); }
    return "";
}

// Every cluster of `fleet` against a new assigner: the same topics, or the same exception text.
static int checkAgainstFreshAssigners(const std::vector<Cluster>& fleet, const std::vector<KafkaTopicAssigner::CandidateResult>& res) {
    CHECK(res.size() == fleet.size());
    int failed = 0;
    for (size_t k = 0; k < fleet.size() && k < res.size(); ++k) {
        KafkaTopicAssigner fresh;
        std::string want;
        std::vector<TopicOutput> exp;
        try { exp = fresh.solveTopics(fleet[k].topics, fleet[k].brokers, fleet[k].rackAssignment, fleet[k].desiredReplicationFactor); }
        catch (const std::exception& e) { want = e.what(); }
        if (want.empty()) {
            CHECK(res[k].status.code == KA_OK);
            CHECK(sameTopics(res[k].topics, exp));
        } else {
            ++failed;
            const std::string got = messageOf(res[k].status, fleet[k].topics);
            if (got != want) { std::fprintf(stderr, "cluster %zu: got '%s' want '%s'\n", k, got.c_str(), want.c_str()); ++failures; }
        }
    }
    return failed;
}

static void testClustersEqualFreshAssigners() {
    const std::vector<Cluster> fleet = {
        cluster(makeTopics(7u, 60, 30), 1, 30, 0),          // no racks
        cluster(makeTopics(8u, 20, 24), 1, 24, 4, 2),       // four racks, RF 2
        cluster(makeTopics(9u, 0, 10), 1, 10, 0),           // no topics
        cluster(makeTopics(10u, 40, 40), 3, 40, 5),         // expansion
        cluster(makeTopics(11u, 30, 30), 1, 2, 0),          // fewer brokers than RF 3: "higher replication factor"
        cluster(makeTopics(12u, 30, 30), 1, 30, 2),         // RF 3 over two racks: "could not be fully assigned"
        cluster(makeTopics(13u, 10, 30), 1, 0, 0),          // no broker at all
        cluster(makeTopics(14u, 50, 30), 5, 30, 3, 1),      // shrinks to RF 1
    };
    KafkaTopicAssigner mine;
    const auto warm = mine.solveTopics(fleet[0].topics, fleet[0].brokers, fleet[0].rackAssignment, -1);   // counters in its Context
    const int failed = checkAgainstFreshAssigners(fleet, mine.solveClusters(fleet));
    CHECK(failed >= 3);
    // the instance's own Context went on as if the batched call had not happened
    KafkaTopicAssigner twice;
    twice.solveTopics(fleet[0].topics, fleet[0].brokers, fleet[0].rackAssignment, -1);
    CHECK(!warm.empty());
    CHECK(sameTopics(mine.solveTopics(fleet[0].topics, fleet[0].brokers, fleet[0].rackAssignment, -1),
                     twice.solveTopics(fleet[0].topics, fleet[0].brokers, fleet[0].rackAssignment, -1)));
}

static void testExceptionTexts() {   // the five reference exceptions, one per cluster, between clusters that solve
    const std::vector<TopicInput> ok = {{"t", {{0, {1, 2, 3}}, {4, {2, 3, 1}}}}};
    const std::vector<TopicInput> mismatch = {{"a", {{0, {1, 2}}}}, {"t", {{0, {1, 2}}, {1, {1}}}}};
    const std::vector<TopicInput> empty = {{"none", {}}};
    const std::vector<TopicInput> minHash = {{"polygenelubricants", {{5, {1, 2, 3}}}}};
    Cluster twoRacks = cluster(ok, 1, 3, 0);
    twoRacks.rackAssignment = {{1, "x"}, {2, "x"}, {3, "y"}};
    const std::vector<Cluster> fleet = {cluster(ok, 1, 3, 0), cluster(mismatch, 1, 3, 0), cluster(ok, 1, 4, 0), cluster(empty, 1, 3, 0),
                                        cluster(ok, 1, 2, 0), twoRacks, cluster(minHash, 1, 3, 0), cluster(ok, 2, 5, 0)};
    KafkaTopicAssigner a;
    const auto res = a.solveClusters(fleet);
    CHECK(checkAgainstFreshAssigners(fleet, res) == 5);
    CHECK(messageOf(res[1].status, mismatch) == "Topic t has partition 1 with unexpected replication factor 1");
    CHECK(res[1].status.topic_index == 1);
    CHECK(messageOf(res[3].status, empty) == "Topic none does not have a positive replication factor!");
    CHECK(messageOf(res[4].status, ok) == "Topic t has a higher replication factor (3) than available brokers!");
    CHECK(messageOf(res[5].status, ok) == "Partition 0 could not be fully assigned!");
    CHECK(messageOf(res[6].status, minHash) == "-2");
    CHECK(res[0].status.code == KA_OK && res[2].status.code == KA_OK && res[7].status.code == KA_OK);
}

int main() {
    try {
        testClustersEqualFreshAssigners();
        testExceptionTexts();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 2;
    }
    std::printf("%s (%d failure%s)\n", failures ? "FAILED" : "OK", failures, failures == 1 ? "" : "s");
    return failures ? 1 : 0;
}
