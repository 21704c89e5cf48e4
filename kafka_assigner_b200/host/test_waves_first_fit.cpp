// test_waves_first_fit.cpp — KafkaTopicAssigner::setWaveRule: planWaves under KA_WAVE_FIRST_FIT over the rows of solveTopics.
// Every changed partition is in exactly one wave; no wave is empty; with unit weights every partition sits in the earliest wave
// where each of its new brokers still has room beside the earlier partitions, and no broker receives more than the budget; the
// device documents of planWavePartsRollback follow the same plan; switching back gives the greedy plan of a fresh instance; an
// unknown rule throws and leaves the rule alone. Needs a GPU (kassign has no CPU fallback). Exit code 0 = all passed.
#include <algorithm>
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

// The wave (1-based) of every (topic, partition) of a plan.
static std::map<std::pair<std::string, int>, int> wavesOf(const KafkaTopicAssigner::WavePlan& plan) {
    std::map<std::pair<std::string, int>, int> res;
    for (size_t v = 0; v < plan.waves.size(); ++v)
        for (const TopicOutput& t : plan.waves[v])
            for (const auto& e : t.assignment) res[{t.name, e.first}] = (int)v + 1;
    return res;
}

int main() {
    const std::vector<TopicInput> topics = makeTopics(11, 400, 30, 12);
    std::set<int> brokers;
    std::map<int, std::string> racks;
    for (int b = 1; b <= 40; ++b) {   // brokers 31..40 joined empty
        brokers.insert(b);
        racks[b] = "rack" + std::to_string(b % 5);
    }
    KafkaTopicAssigner a;
    const std::vector<TopicOutput> proposed = a.solveTopics(topics, brokers, racks, -1);
    CHECK(a.waveRule() == KA_WAVE_GREEDY);
    const KafkaTopicAssigner::WavePlan greedy = a.planWaves(topics, proposed, 2);
    a.setWaveRule(KA_WAVE_FIRST_FIT);
    CHECK(a.waveRule() == KA_WAVE_FIRST_FIT);
    bool threw = false;
    try {
        a.setWaveRule(7);
    } catch (const kassign::KassignError& e) {
        threw = e.code == KA_ERR_BAD_ARG;
    }
    CHECK(threw && a.waveRule() == KA_WAVE_FIRST_FIT);

    for (const int64_t budget : {1, 2, 5}) {
        const KafkaTopicAssigner::WavePlan plan = a.planWaves(topics, proposed, budget);
        CHECK(plan.status.code == KA_OK && !plan.waves.empty() && plan.waves.size() == plan.summary.size());
        const auto wave = wavesOf(plan);
        // in input order, each changed partition's wave is the first where every new broker has room
        std::map<std::pair<int, int>, int64_t> in;   // (broker, wave) -> partitions received
        int changed = 0;
        for (size_t t = 0; t < topics.size(); ++t)
            for (const auto& e : proposed[t].assignment) {
                const std::vector<int>& cur = topics[t].current.at(e.first);
                if (e.second == cur) {
                    CHECK(!wave.count({topics[t].name, e.first}));
                    continue;
                }
                ++changed;
                std::vector<int> recv;
                for (int b : e.second)
                    if (std::find(cur.begin(), cur.end(), b) == cur.end()) recv.push_back(b);
                int v = 1;
                if (!recv.empty())
                    while (std::any_of(recv.begin(), recv.end(), [&](int b) { return in[{b, v}] + 1 > budget; })) ++v;
                CHECK(wave.at({topics[t].name, e.first}) == v);
                for (int b : recv) ++in[{b, v}];
            }
        CHECK((int)wave.size() == changed && changed > 50);
        for (size_t v = 0; v < plan.waves.size(); ++v) {
            int64_t rows = 0, peak = 0;
            for (const TopicOutput& t : plan.waves[v]) rows += (int64_t)t.assignment.size();
            for (const auto& e : in)
                if (e.first.second == (int)v + 1) peak = std::max(peak, e.second);
            CHECK(rows == plan.summary[v].rows && rows > 0 && peak == plan.summary[v].max_broker_in && peak <= budget);
        }
        // the device documents follow the same plan
        const KafkaTopicAssigner::WaveRollback docs = a.planWavePartsRollback(topics, proposed, budget, 1 << 20);
        CHECK(docs.status.code == KA_OK && docs.parts.size() == plan.waves.size());
        for (size_t v = 0; v < docs.parts.size() && v < plan.waves.size(); ++v)
            CHECK(docs.parts[v] == kassign::newAssignmentJson(plan.waves[v]) && docs.partWave[v] == (int)v + 1);
    }
    a.setWaveRule(KA_WAVE_GREEDY);
    const KafkaTopicAssigner::WavePlan back = a.planWaves(topics, proposed, 2);
    CHECK(back.status.code == KA_OK && wavesOf(back) == wavesOf(greedy) && back.waves.size() == greedy.waves.size());
    if (failures) {
        std::printf("FAILED %d\n", failures);
        return 1;
    }
    std::printf("OK\n");
    return 0;
}
