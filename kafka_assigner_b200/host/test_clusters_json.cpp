// test_clusters_json.cpp — KafkaTopicAssigner::solveClustersJson against the per-cluster runs it replaces: every cluster's
// text equals solveTopicsJson on a new KafkaTopicAssigner with its own broker set and desired replication factor, a failing
// cluster re-throws the reference's message text without touching the others, and the clusters the device call refuses
// (names that need escapes, rows wider than 3) still get the text solveTopicsJson gives them. Needs a GPU (kassign has no CPU
// fallback). Exit code 0 = all passed.
#include <cstdio>
#include <cstdlib>

#include "kassign_host.hpp"

using kassign::KafkaTopicAssigner;
using kassign::TopicInput;
using Cluster = KafkaTopicAssigner::ClusterInput;

static int failures = 0;
#define CHECK(cond)                                                              \
    do {                                                                         \
        if (!(cond)) { std::fprintf(stderr, "FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); ++failures; } \
    } while (0)

// A seeded ragged run: 1..40 partitions per topic with sparse ids, replication factor 1..rfmax, lists on brokers 1..nb.
static std::vector<TopicInput> makeTopics(unsigned seed, int T, int nb, int rfmax = 3, const std::string& prefix = "svc.topic-") {
    auto next = [&]() { seed = seed * 1103515245u + 12345u; return (int)((seed >> 8) & 0xFFFF); };
    std::vector<TopicInput> topics(T);
    for (int t = 0; t < T; ++t) {
        topics[t].name = prefix + std::to_string(t);
        const int P = 1 + next() % 40, rf = 1 + next() % rfmax;
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

// Every cluster of `fleet` against a new assigner: the same text, or the same exception text. Returns the failed clusters.
static int checkAgainstFreshAssigners(const std::vector<Cluster>& fleet, const std::vector<KafkaTopicAssigner::ClusterJson>& res) {
    CHECK(res.size() == fleet.size());
    int failed = 0;
    for (size_t k = 0; k < fleet.size() && k < res.size(); ++k) {
        KafkaTopicAssigner fresh;
        std::string want, exp;
        try { exp = fresh.solveTopicsJson(fleet[k].topics, fleet[k].brokers, fleet[k].rackAssignment, fleet[k].desiredReplicationFactor); }
        catch (const std::exception& e) { want = e.what(); }
        if (want.empty()) {
            CHECK(res[k].status.code == KA_OK);
            if (res[k].json != exp) { std::fprintf(stderr, "cluster %zu: text differs\n", k); ++failures; }
        } else {
            ++failed;
            CHECK(res[k].json.empty());
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
    const std::string warm = mine.solveTopicsJson(fleet[0].topics, fleet[0].brokers, fleet[0].rackAssignment, -1);   // counters in its Context
    CHECK(checkAgainstFreshAssigners(fleet, mine.solveClustersJson(fleet)) >= 3);
    // the instance's own Context went on as if the batched call had not happened
    KafkaTopicAssigner twice;
    twice.solveTopicsJson(fleet[0].topics, fleet[0].brokers, fleet[0].rackAssignment, -1);
    CHECK(!warm.empty());
    CHECK(mine.solveTopicsJson(fleet[0].topics, fleet[0].brokers, fleet[0].rackAssignment, -1) ==
          twice.solveTopicsJson(fleet[0].topics, fleet[0].brokers, fleet[0].rackAssignment, -1));
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
    const auto res = a.solveClustersJson(fleet);
    CHECK(checkAgainstFreshAssigners(fleet, res) == 5);
    CHECK(messageOf(res[1].status, mismatch) == "Topic t has partition 1 with unexpected replication factor 1");
    CHECK(messageOf(res[3].status, empty) == "Topic none does not have a positive replication factor!");
    CHECK(messageOf(res[4].status, ok) == "Topic t has a higher replication factor (3) than available brokers!");
    CHECK(messageOf(res[5].status, ok) == "Partition 0 could not be fully assigned!");
    CHECK(messageOf(res[6].status, minHash) == "-2");
    CHECK(res[0].json.rfind("{\"partitions\":[{\"partition\":0,", 0) == 0);
}

// The clusters the device call refuses: a name org.json escapes (host emitter) and rows of 4 and 5 (the fused chain of
// ka_solve_json), next to clusters the device call solves.
static void testFallbacks() {
    std::vector<TopicInput> quoted = makeTopics(21u, 12, 20);
    quoted[3].name = "a\"b</c";
    const std::vector<Cluster> fleet = {
        cluster(makeTopics(20u, 30, 30), 1, 30, 0),
        cluster(quoted, 1, 20, 0),
        cluster(makeTopics(22u, 25, 40, 4), 1, 40, 0),             // lists of up to 4
        cluster(makeTopics(23u, 25, 40, 5, "wide-"), 1, 40, 0),    // lists of up to 5
        cluster(makeTopics(24u, 30, 30), 1, 30, 0),
    };
    KafkaTopicAssigner a;
    const auto res = a.solveClustersJson(fleet);
    CHECK(checkAgainstFreshAssigners(fleet, res) == 0);
    for (size_t k = 0; k < res.size(); ++k)
        if (res[k].status.code != KA_OK) std::fprintf(stderr, "cluster %zu: status %d a=%d\n", k, res[k].status.code, res[k].status.a);
    CHECK(res[1].json.find("\"topic\":\"a\\\"b<\\/c\"") != std::string::npos);
    CHECK(res[2].json.find("\"replicas\":[") != std::string::npos);
}

int main() {
    try {
        testClustersEqualFreshAssigners();
        testExceptionTexts();
        testFallbacks();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 2;
    }
    std::printf("%s (%d failure%s)\n", failures ? "FAILED" : "OK", failures, failures == 1 ? "" : "s");
    return failures ? 1 : 0;
}
