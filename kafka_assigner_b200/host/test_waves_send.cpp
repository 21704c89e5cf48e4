// test_waves_send.cpp — the SendBudget overloads of KafkaTopicAssigner::planWaves / planWavesJson over the rows of solveTopics
// with a drained broker: in every wave no broker receives more than the receive budget and no partition leader (the first broker
// of its current list) sends more than the send budget, unless one partition alone exceeds it; the documents of planWavesJson
// equal newAssignmentJson of the same waves; with a send budget no plan reaches and no leader moving two partitions, both equal
// the calls without one; a leader
// missing from the send table is refused with its row and id. Needs a GPU (kassign has no CPU fallback). Exit code 0 = all
// passed.
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

// The seeded ragged run of test_waves.cpp: 1..maxP partitions per topic with sparse ids, replication factor 1..3, lists on
// brokers 1..nb.
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

// Both budgets over the waves of a plan with unit weights: per wave, what each broker receives (new-list brokers the current
// list lacks) and what each leader sends (its partition's receivers) stays within the budget, or comes from one partition alone.
static void checkBudgets(const std::vector<TopicInput>& topics, const KafkaTopicAssigner::WavePlan& plan, int64_t maxIn,
                         int64_t maxOut) {
    for (const std::vector<TopicOutput>& wave : plan.waves) {
        std::map<int, std::pair<int64_t, int>> in, out;   // broker -> (sum, partitions adding to it)
        for (const TopicOutput& t : wave) {
            const TopicInput* src = nullptr;
            for (const TopicInput& x : topics)
                if (x.name == t.name) src = &x;
            CHECK(src != nullptr);
            if (!src) continue;
            for (const auto& e : t.assignment) {
                const std::vector<int>& cur = src->current.at(e.first);
                int r = 0;
                for (int b : e.second)
                    if (std::find(cur.begin(), cur.end(), b) == cur.end()) {
                        ++r;
                        in[b].first += 1;
                        in[b].second += 1;
                    }
                if (r > 0 && !cur.empty()) {
                    out[cur[0]].first += r;
                    out[cur[0]].second += 1;
                }
            }
        }
        for (const auto& x : in) CHECK(x.second.first <= maxIn || x.second.second == 1);
        for (const auto& x : out) CHECK(x.second.first <= maxOut || x.second.second == 1);
    }
}

int main() {
    const std::vector<TopicInput> topics = makeTopics(11, 400, 30, 12);
    std::set<int> brokers;
    std::map<int, std::string> racks;
    std::vector<int32_t> everyBroker;
    for (int b = 1; b <= 40; ++b) {   // broker 3 is drained; brokers 31..40 joined empty
        everyBroker.push_back(b);
        if (b == 3) continue;
        brokers.insert(b);
        racks[b] = "rack" + std::to_string(b % 5);
    }
    KafkaTopicAssigner a;
    const std::vector<TopicOutput> proposed = a.solveTopics(topics, brokers, racks, -1);

    for (const int64_t maxIn : {2, 8}) {
        const KafkaTopicAssigner::WavePlan open = a.planWaves(topics, proposed, maxIn);
        for (const int64_t maxOut : {3, 6, 20}) {
            const KafkaTopicAssigner::SendBudget send{maxOut, everyBroker};
            const KafkaTopicAssigner::WavePlan plan = a.planWaves(topics, proposed, maxIn, send);
            CHECK(plan.status.code == KA_OK && !plan.waves.empty());
            CHECK(plan.sendSummary.size() == plan.summary.size() && plan.waves.size() >= open.waves.size());
            checkBudgets(topics, plan, maxIn, maxOut);
            for (const ka_wave_send_summary& s : plan.sendSummary) CHECK(s.max_broker_out <= maxOut);
            const KafkaTopicAssigner::WaveDocs docs = a.planWavesJson(topics, proposed, maxIn, send);
            CHECK(docs.status.code == KA_OK && docs.docs.size() == plan.waves.size());
            for (size_t v = 0; v < plan.waves.size() && v < docs.docs.size(); ++v) {
                CHECK(docs.docs[v] == kassign::newAssignmentJson(plan.waves[v]));
                CHECK(std::memcmp(&docs.summary[v], &plan.summary[v], sizeof(ka_wave_summary)) == 0);
                CHECK(std::memcmp(&docs.sendSummary[v], &plan.sendSummary[v], sizeof(ka_wave_send_summary)) == 0);
            }
        }
    }

    // a send budget no plan reaches, where no leader has two moved partitions: the plan and the documents of the calls without one
    std::vector<TopicInput> uniq(1);
    std::vector<TopicOutput> uniqProposed(1);
    uniq[0].name = uniqProposed[0].name = "uniq";
    for (int p = 0; p < 35; ++p) {   // partition p led by broker p + 1, each gaining one of brokers 36..40
        uniq[0].current[p] = {p + 1};
        uniqProposed[0].assignment[p] = {p + 1, 36 + p % 5};
    }
    for (const int64_t maxIn : {1, 3}) {
        const KafkaTopicAssigner::SendBudget huge{INT64_MAX, everyBroker};
        const KafkaTopicAssigner::WavePlan open = a.planWaves(uniq, uniqProposed, maxIn);
        const KafkaTopicAssigner::WavePlan same = a.planWaves(uniq, uniqProposed, maxIn, huge);
        CHECK(same.status.code == KA_OK && same.waves.size() == open.waves.size() && same.summary.size() == open.summary.size());
        CHECK(open.waves.size() == (maxIn == 1 ? 7u : 3u));
        for (size_t v = 0; v < same.waves.size() && v < open.waves.size(); ++v) {
            CHECK(kassign::newAssignmentJson(same.waves[v]) == kassign::newAssignmentJson(open.waves[v]));
            CHECK(std::memcmp(&same.summary[v], &open.summary[v], sizeof(ka_wave_summary)) == 0);
        }
        const KafkaTopicAssigner::WaveDocs sameDocs = a.planWavesJson(uniq, uniqProposed, maxIn, huge);
        const KafkaTopicAssigner::WaveDocs openDocs = a.planWavesJson(uniq, uniqProposed, maxIn);
        CHECK(sameDocs.status.code == KA_OK && sameDocs.docs == openDocs.docs);
    }

    // a leader the send table lacks: refused with the first such row and the leader's id
    std::vector<int32_t> live(brokers.begin(), brokers.end());
    const KafkaTopicAssigner::WavePlan refused = a.planWaves(topics, proposed, 4, KafkaTopicAssigner::SendBudget{4, live});
    CHECK(refused.status.code == KA_ERR_BAD_ARG && refused.status.b == 3 && refused.waves.empty() && refused.sendSummary.empty());
    const KafkaTopicAssigner::WaveDocs refusedDocs = a.planWavesJson(topics, proposed, 4, KafkaTopicAssigner::SendBudget{4, live});
    CHECK(refusedDocs.status.code == KA_ERR_BAD_ARG && refusedDocs.status.b == 3 && refusedDocs.status.a == refused.status.a);
    if (failures) {
        std::printf("FAILED %d\n", failures);
        return 1;
    }
    std::printf("OK\n");
    return 0;
}
