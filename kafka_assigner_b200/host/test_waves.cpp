// test_waves.cpp — KafkaTopicAssigner::planWaves over the rows of solveTopics: the documents of all waves (newAssignmentJson of
// each wave), taken together, hold exactly the changed partitions of newAssignmentJson(solveTopics(...)), one record each; every
// wave's summary counts its records; with unit weights no broker receives more than the budget in a wave; a refused proposal
// carries its status. Needs a GPU (kassign has no CPU fallback). Exit code 0 = all passed.
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

// The partition records of an org.json document, in document order.
static std::vector<std::string> records(const std::string& json) {
    std::vector<std::string> res;
    for (size_t at = json.find("{\"partition\":"); at != std::string::npos; at = json.find("{\"partition\":", at + 1))
        res.push_back(json.substr(at, json.find('}', at) - at + 1));
    return res;
}

int main() {
    const std::vector<TopicInput> topics = makeTopics(7, 400, 30, 12);
    std::set<int> brokers;
    std::map<int, std::string> racks;
    for (int b = 1; b <= 40; ++b) {   // brokers 31..40 joined empty
        brokers.insert(b);
        racks[b] = "rack" + std::to_string(b % 5);
    }
    KafkaTopicAssigner a;
    const std::vector<TopicOutput> proposed = a.solveTopics(topics, brokers, racks, -1);
    // the changed partitions, as records of the full document
    std::vector<TopicOutput> changed;
    int nChanged = 0;
    for (size_t t = 0; t < topics.size(); ++t) {
        changed.push_back(TopicOutput{topics[t].name, {}});
        for (const auto& e : proposed[t].assignment)
            if (e.second != topics[t].current.at(e.first)) {
                changed.back().assignment[e.first] = e.second;
                ++nChanged;
            }
    }
    std::vector<std::string> want = records(kassign::newAssignmentJson(changed));
    const std::vector<std::string> all = records(kassign::newAssignmentJson(proposed));
    CHECK(nChanged > 50 && (int)want.size() == nChanged);
    for (const std::string& r : want) CHECK(std::find(all.begin(), all.end(), r) != all.end());
    std::sort(want.begin(), want.end());

    std::vector<std::map<int, int64_t>> weights(topics.size());
    unsigned seed = 3;
    for (size_t t = 0; t < topics.size(); ++t)
        for (const auto& p : topics[t].current) { seed = seed * 1103515245u + 12345u; weights[t][p.first] = (seed >> 8) % 100; }
    struct Case { int64_t budget; bool weighted; };
    for (const Case c : {Case{1, false}, Case{4, false}, Case{1000000, false}, Case{150, true}, Case{1, true}}) {
        const KafkaTopicAssigner::WavePlan plan = a.planWaves(topics, proposed, c.budget, c.weighted ? weights : std::vector<std::map<int, int64_t>>{});
        CHECK(plan.status.code == KA_OK);
        CHECK(plan.waves.size() == plan.summary.size() && !plan.waves.empty());
        if (c.budget == 1000000) CHECK(plan.waves.size() == 1);
        std::vector<std::string> got;
        for (size_t v = 0; v < plan.waves.size(); ++v) {
            const std::vector<std::string> rec = records(kassign::newAssignmentJson(plan.waves[v]));
            CHECK((int64_t)rec.size() == plan.summary[v].rows && !rec.empty());
            got.insert(got.end(), rec.begin(), rec.end());
            if (c.weighted) continue;
            std::map<int, int64_t> in;   // unit weights: every broker receives at most the budget in the wave
            for (const TopicOutput& t : plan.waves[v]) {
                const auto& cur = std::find_if(topics.begin(), topics.end(), [&](const TopicInput& x) { return x.name == t.name; })->current;
                for (const auto& e : t.assignment)
                    for (int b : e.second)
                        if (std::find(cur.at(e.first).begin(), cur.at(e.first).end(), b) == cur.at(e.first).end()) ++in[b];
            }
            int64_t peak = 0;
            for (const auto& e : in) peak = std::max(peak, e.second);
            CHECK(peak <= c.budget && peak == plan.summary[v].max_broker_in);
        }
        std::sort(got.begin(), got.end());
        CHECK(got == want);
    }
    // a proposal naming a broker twice is refused with its row and broker
    std::vector<TopicOutput> bad = proposed;
    bad[2].assignment.begin()->second = {7, 7};
    const KafkaTopicAssigner::WavePlan refused = a.planWaves(topics, bad, 3);
    CHECK(refused.status.code == KA_ERR_BAD_ARG && refused.status.b == 7 && refused.waves.empty() && refused.summary.empty());
    CHECK(refused.status.a == (int)(topics[0].current.size() + topics[1].current.size()));
    if (failures) {
        std::printf("FAILED %d\n", failures);
        return 1;
    }
    std::printf("OK\n");
    return 0;
}
