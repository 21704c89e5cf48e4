// test_candidates.cpp — KafkaTopicAssigner::solveTopicsCandidates against the per-candidate runs it replaces: every
// candidate equals solveTopics on a new KafkaTopicAssigner with that broker set, a failing candidate re-throws the
// reference's message text (KTA:58-60, 65-66, 67-69; KAS:183-184), and the instance's own Context is left alone.
// Needs a GPU (kassign has no CPU fallback). Exit code 0 = all passed.
#include <cstdio>
#include <cstdlib>

#include "kassign_host.hpp"

using kassign::KafkaTopicAssigner;
using kassign::TopicInput;
using kassign::TopicOutput;

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

static KafkaTopicAssigner::Candidate candidate(int lo, int hi, int racks) {
    KafkaTopicAssigner::Candidate c;
    for (int b = lo; b <= hi; ++b) {
        c.brokers.insert(b);
        if (racks > 0) c.rackAssignment[b] = "rack" + std::to_string(b % racks);
    }
    return c;
}

static std::string messageOf(const ka_status& st, const std::vector<TopicInput>& topics) {
    std::vector<std::string> names;
    for (const auto& t : topics) names.push_back(t.name);
    try { kassign::throwForStatus(st, names); } catch (const std::exception& e) { return e.what(); }
    return "";
}

static void testCandidatesEqualFreshAssigners() {
    const std::vector<TopicInput> topics = makeTopics(7u, 60, 30);
    std::vector<KafkaTopicAssigner::Candidate> cands = {
        candidate(1, 30, 0),    // every broker, no racks
        candidate(1, 24, 0),    // decommission
        candidate(1, 30, 4),    // every broker in four racks
        candidate(3, 40, 5),    // expansion
        candidate(1, 2, 0),     // fewer brokers than RF 3: "higher replication factor"
        candidate(1, 30, 2),    // RF 3 over two racks: "could not be fully assigned"
        candidate(1, 0, 0),     // no broker at all
        candidate(5, 30, 3),
    };
    // a run through an assigner's own Context; a failed run gives no topics
    auto run = [&](KafkaTopicAssigner& a, const KafkaTopicAssigner::Candidate& c) {
        try { return a.solveTopics(topics, c.brokers, c.rackAssignment, -1); } catch (const std::exception&) { return std::vector<TopicOutput>(); }
    };
    KafkaTopicAssigner mine;
    const auto warm = run(mine, cands[0]);   // counters in its Context
    for (int desired : {-1, 2, 3}) {
        const auto res = mine.solveTopicsCandidates(topics, cands, desired);
        CHECK(res.size() == cands.size());
        int failed = 0;
        for (size_t k = 0; k < cands.size(); ++k) {
            KafkaTopicAssigner fresh;
            std::string want;
            std::vector<TopicOutput> exp;
            try { exp = fresh.solveTopics(topics, cands[k].brokers, cands[k].rackAssignment, desired); }
            catch (const std::exception& e) { want = e.what(); }
            if (want.empty()) {
                CHECK(res[k].status.code == KA_OK);
                CHECK(sameTopics(res[k].topics, exp));
            } else {
                ++failed;
                if (messageOf(res[k].status, topics) != want)
                    { std::fprintf(stderr, "candidate %zu: got '%s' want '%s'\n", k, messageOf(res[k].status, topics).c_str(), want.c_str()); ++failures; }
            }
        }
        CHECK(failed >= (desired == 2 ? 1 : 3));
    }
    // the instance's own Context went on as if the batched calls had not happened
    KafkaTopicAssigner twice;
    run(twice, cands[0]);
    CHECK(!warm.empty());
    CHECK(sameTopics(run(mine, cands[0]), run(twice, cands[0])));
}

static void testExceptionTexts() {   // one reference exception per candidate of one call
    const std::vector<TopicInput> topics = {{"t", {{0, {1, 2}}, {1, {1}}}}};
    const std::vector<TopicInput> ok = {{"t", {{0, {1, 2, 3}}, {4, {2, 3, 1}}}}};
    KafkaTopicAssigner a;
    auto res = a.solveTopicsCandidates(topics, {candidate(1, 3, 0)}, -1);
    CHECK(messageOf(res[0].status, topics) == "Topic t has partition 1 with unexpected replication factor 1");
    res = a.solveTopicsCandidates(ok, {candidate(1, 3, 0), candidate(1, 2, 0), candidate(1, 3, 0)}, -1);
    CHECK(res[0].status.code == KA_OK && res[2].status.code == KA_OK);
    CHECK(messageOf(res[1].status, ok) == "Topic t has a higher replication factor (3) than available brokers!");
    KafkaTopicAssigner::Candidate twoRacks = candidate(1, 3, 0);
    twoRacks.rackAssignment = {{1, "x"}, {2, "x"}, {3, "y"}};
    res = a.solveTopicsCandidates(ok, {candidate(1, 4, 0), twoRacks}, -1);
    CHECK(res[0].status.code == KA_OK);
    CHECK(messageOf(res[1].status, ok) == "Partition 0 could not be fully assigned!");
    const std::vector<TopicInput> empty = {{"none", {}}};
    res = a.solveTopicsCandidates(empty, {candidate(1, 3, 0)}, -1);
    CHECK(messageOf(res[0].status, empty) == "Topic none does not have a positive replication factor!");
    const std::vector<TopicInput> minHash = {{"polygenelubricants", {{5, {1, 2, 3}}}}};
    res = a.solveTopicsCandidates(minHash, {candidate(1, 3, 0)}, -1);
    CHECK(messageOf(res[0].status, minHash) == "-2");
}

int main() {
    try {
        testCandidatesEqualFreshAssigners();
        testExceptionTexts();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 2;
    }
    std::printf("%s (%d failure%s)\n", failures ? "FAILED" : "OK", failures, failures == 1 ? "" : "s");
    return failures ? 1 : 0;
}
