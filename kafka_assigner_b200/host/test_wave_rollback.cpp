// test_wave_rollback.cpp — KafkaTopicAssigner::planWavePartsRollback over the rows of solveTopics: every rollback document is
// kafkaReassignmentJson of its part's partitions (in the part's order, on their current lists); both sides are within the
// limit and a part could not take the next part's first partition on both; without a longer current list the parts are those
// of planWaveParts; names that org.json escapes take the host cut and give what the device gives for names of the same
// length; an over-long partition and a refused proposal carry their status.
// Needs a GPU (kassign has no CPU fallback). Exit code 0 = all passed.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "kassign_host.hpp"

using kassign::KafkaTopicAssigner;
using kassign::TopicInput;
using kassign::TopicOutput;

static int failures = 0;
#define CHECK(cond)                                                              \
    do {                                                                         \
        if (!(cond)) { std::fprintf(stderr, "FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); ++failures; } \
    } while (0)

// A seeded ragged run with RF 1..rfMax current lists.
static std::vector<TopicInput> makeTopics(unsigned seed, int T, int nb, int maxP, int rfMax, const std::string& stem) {
    auto next = [&]() { seed = seed * 1103515245u + 12345u; return (int)((seed >> 8) & 0xFFFF); };
    std::vector<TopicInput> topics(T);
    for (int t = 0; t < T; ++t) {
        topics[t].name = stem + std::to_string(t);
        const int P = 1 + next() % maxP, rf = 1 + next() % rfMax;
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

// The (topic, partition) of every record of a forward document, in order; topic names here hold no '"'.
static std::vector<std::pair<std::string, int>> keys(const std::string& doc) {
    std::vector<std::pair<std::string, int>> out;
    for (size_t at = doc.find("{\"partition\":"); at != std::string::npos; at = doc.find("{\"partition\":", at + 1)) {
        const int part = std::atoi(doc.c_str() + at + 13);
        const size_t name = doc.find("\"topic\":\"", at) + 9;
        out.emplace_back(doc.substr(name, doc.find('"', name) - name), part);
    }
    return out;
}

// kafkaReassignmentJson of these partitions, in this order, on their current lists.
static std::string rollbackOf(const std::vector<TopicInput>& topics, const std::vector<std::pair<std::string, int>>& ks) {
    std::vector<TopicInput> in;
    for (const auto& k : ks) {
        if (in.empty() || in.back().name != k.first) in.push_back(TopicInput{k.first, {}});
        for (const TopicInput& t : topics)
            if (t.name == k.first) in.back().current[k.second] = t.current.at(k.second);
    }
    return kafkaReassignmentJson(in);
}

static void compare(KafkaTopicAssigner& a, const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed,
                    int64_t budget, int64_t limit, const std::vector<std::map<int, int64_t>>& weights,
                    const KafkaTopicAssigner::SendBudget* send, bool longerCurrent) {
    const KafkaTopicAssigner::WaveParts parts = send ? a.planWaveParts(topics, proposed, budget, limit, *send, weights)
                                                     : a.planWaveParts(topics, proposed, budget, limit, weights);
    const KafkaTopicAssigner::WaveRollback rb = send ? a.planWavePartsRollback(topics, proposed, budget, limit, *send, weights)
                                                     : a.planWavePartsRollback(topics, proposed, budget, limit, weights);
    CHECK(parts.status.code == KA_OK && rb.status.code == KA_OK);
    CHECK(rb.summary.size() == parts.summary.size() && rb.parts.size() == rb.partWave.size() && rb.parts.size() == rb.rollback.size());
    CHECK(std::memcmp(rb.summary.data(), parts.summary.data(), parts.summary.size() * sizeof(ka_wave_summary)) == 0);
    if (send) CHECK(std::memcmp(rb.sendSummary.data(), parts.sendSummary.data(), parts.sendSummary.size() * sizeof(ka_wave_send_summary)) == 0);
    if (!longerCurrent) CHECK(rb.parts == parts.parts && rb.partWave == parts.partWave);
    else CHECK(rb.parts.size() >= parts.parts.size());
    for (size_t d = 0; d < rb.parts.size(); ++d) {
        CHECK((int64_t)rb.parts[d].size() <= limit && (int64_t)rb.rollback[d].size() <= limit);
        const auto ks = keys(rb.parts[d]);
        CHECK(rb.rollback[d] == rollbackOf(topics, ks));
        if (d + 1 < rb.parts.size() && rb.partWave[d + 1] == rb.partWave[d]) {   // the next part's first partition fits on no side
            auto more = ks;
            more.push_back(keys(rb.parts[d + 1]).front());
            const std::string& next = rb.parts[d + 1];
            const size_t end = next.find("},{");
            const size_t first = (end == std::string::npos ? next.size() - 14 : end + 1) - 15;   // its first record
            CHECK((int64_t)rollbackOf(topics, more).size() > limit || (int64_t)(rb.parts[d].size() + 1 + first) > limit);
        }
    }
}

int main() {
    std::set<int> brokers;
    std::map<int, std::string> racks;
    for (int b = 1; b <= 40; ++b) {   // brokers 31..40 joined empty
        brokers.insert(b);
        racks[b] = "rack" + std::to_string(b % 5);
    }
    KafkaTopicAssigner a;
    // RF 1..3 solved to RF 2: the RF-3 topics shrink, their rollback records are the longer side
    const std::vector<TopicInput> topics = makeTopics(7, 300, 30, 12, 3, "svc.topic-");
    const std::vector<TopicOutput> shrunk = a.solveTopics(topics, brokers, racks, 2);
    // RF 1..2 on brokers 1..9 solved to RF 3: every proposed list has more brokers, of as many digits or more, so no rollback
    // record is longer than its forward record
    const std::vector<TopicInput> small = makeTopics(9, 300, 9, 12, 2, "svc.grow-");
    const std::vector<TopicOutput> grown = a.solveTopics(small, brokers, racks, 3);
    std::vector<std::map<int, int64_t>> weights(topics.size());
    unsigned seed = 3;
    for (size_t t = 0; t < topics.size(); ++t)
        for (const auto& p : topics[t].current) { seed = seed * 1103515245u + 12345u; weights[t][p.first] = (seed >> 8) % 100; }
    KafkaTopicAssigner::SendBudget send{3, {}};
    for (int b = 1; b <= 40; ++b) send.sendBrokers.push_back(b);
    for (const int64_t limit : {120, 250, 4096, 1 << 20}) {
        for (const int64_t budget : {1, 4, 1000000}) compare(a, topics, shrunk, budget, limit, {}, nullptr, true);
        compare(a, topics, shrunk, 150, limit, weights, nullptr, true);
        compare(a, topics, shrunk, 2, limit, {}, &send, true);
    }
    for (const int64_t limit : {120, 1000, 1 << 20}) {
        compare(a, small, grown, 3, limit, {}, nullptr, false);
        compare(a, small, grown, 2, limit, {}, &send, false);
    }

    // names org.json escapes ('/', printed as is): the host cut gives what the device gives for names of the same length
    std::vector<TopicInput> odd = topics;
    std::vector<TopicOutput> oddProposed = shrunk;
    for (size_t t = 0; t < odd.size(); ++t) odd[t].name = oddProposed[t].name = "svc/topic-" + std::to_string(t);
    for (const int64_t limit : {120, 1000, 1 << 20}) {
        compare(a, odd, oddProposed, 2, limit, {}, nullptr, true);
        const KafkaTopicAssigner::WaveRollback host = a.planWavePartsRollback(odd, oddProposed, 2, limit);
        const KafkaTopicAssigner::WaveRollback dev = a.planWavePartsRollback(topics, shrunk, 2, limit);
        CHECK(host.partWave == dev.partWave && host.parts.size() == dev.parts.size());
        for (size_t d = 0; d < host.parts.size() && d < dev.parts.size(); ++d) {
            std::string p = host.parts[d], r = host.rollback[d];
            std::replace(p.begin(), p.end(), '/', '.');
            std::replace(r.begin(), r.end(), '/', '.');
            CHECK(p == dev.parts[d] && r == dev.rollback[d]);
        }
    }

    // a partition whose one-record document on either side exceeds the limit: its row and the longer length, on both paths
    const std::vector<TopicInput>* inputs[] = {&topics, &odd};
    for (const auto* in : inputs) {
        const std::vector<TopicOutput>& prop = in == &topics ? shrunk : oddProposed;
        const KafkaTopicAssigner::WaveRollback tiny = a.planWavePartsRollback(*in, prop, 1000000, 40);
        CHECK(tiny.status.code == KA_ERR_LIMIT && tiny.status.b > 40 && tiny.parts.empty() && tiny.rollback.empty() && tiny.summary.empty());
        const KafkaTopicAssigner::WaveRollback dev = a.planWavePartsRollback(topics, shrunk, 1000000, 40);
        CHECK(tiny.status.a == dev.status.a && tiny.status.b == dev.status.b);
    }

    // nothing changed: no part; a limit below 1 and a refused proposal carry their status
    std::vector<TopicOutput> same;
    for (const TopicInput& t : topics) same.push_back(TopicOutput{t.name, t.current});
    const KafkaTopicAssigner::WaveRollback none = a.planWavePartsRollback(topics, same, 1, 1000);
    CHECK(none.status.code == KA_OK && none.parts.empty() && none.rollback.empty() && none.summary.empty());
    CHECK(a.planWavePartsRollback(topics, shrunk, 1, 0).status.code == KA_ERR_BAD_ARG);
    std::vector<TopicOutput> bad = shrunk;
    bad[2].assignment.begin()->second = {7, 7};
    const KafkaTopicAssigner::WaveRollback refused = a.planWavePartsRollback(topics, bad, 3, 1000);
    CHECK(refused.status.code == KA_ERR_BAD_ARG && refused.status.b == 7 && refused.parts.empty() && refused.rollback.empty());
    if (failures) {
        std::printf("FAILED %d\n", failures);
        return 1;
    }
    std::printf("OK\n");
    return 0;
}
