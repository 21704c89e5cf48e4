// test_waves_json.cpp — KafkaTopicAssigner::planWavesJson over the rows of solveTopics: every document built on the device equals
// newAssignmentJson of the same wave of planWaves, byte for byte, with the same summaries, unit and weighted; topic names that
// org.json escapes take the host emitter and give the same text (with argv[1], a file of such names and their quotes, every one of
// them); a refused proposal carries its status. Needs a GPU (kassign has no CPU fallback). Exit code 0 = all passed.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>

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

static void compare(KafkaTopicAssigner& a, const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed,
                    int64_t budget, const std::vector<std::map<int, int64_t>>& weights) {
    const KafkaTopicAssigner::WavePlan plan = a.planWaves(topics, proposed, budget, weights);
    const KafkaTopicAssigner::WaveDocs docs = a.planWavesJson(topics, proposed, budget, weights);
    CHECK(plan.status.code == KA_OK && docs.status.code == KA_OK);
    CHECK(!plan.waves.empty() && docs.docs.size() == plan.waves.size() && docs.summary.size() == plan.summary.size());
    for (size_t v = 0; v < plan.waves.size() && v < docs.docs.size(); ++v) {
        CHECK(docs.docs[v] == kassign::newAssignmentJson(plan.waves[v]));
        CHECK(std::memcmp(&docs.summary[v], &plan.summary[v], sizeof(ka_wave_summary)) == 0);
    }
}

static std::string unhex(const std::string& h) {
    std::string s;
    for (size_t i = 0; i + 1 < h.size(); i += 2) s.push_back((char)std::stoi(h.substr(i, 2), nullptr, 16));
    return s;
}

int main(int argc, char** argv) {
    std::vector<TopicInput> topics = makeTopics(7, 400, 30, 12);
    std::set<int> brokers;
    std::map<int, std::string> racks;
    for (int b = 1; b <= 40; ++b) {   // brokers 31..40 joined empty
        brokers.insert(b);
        racks[b] = "rack" + std::to_string(b % 5);
    }
    KafkaTopicAssigner a;
    const std::vector<TopicOutput> proposed = a.solveTopics(topics, brokers, racks, -1);
    std::vector<std::map<int, int64_t>> weights(topics.size());
    unsigned seed = 3;
    for (size_t t = 0; t < topics.size(); ++t)
        for (const auto& p : topics[t].current) { seed = seed * 1103515245u + 12345u; weights[t][p.first] = (seed >> 8) % 100; }
    for (const int64_t budget : {1, 4, 1000000}) compare(a, topics, proposed, budget, {});
    for (const int64_t budget : {150, 1}) compare(a, topics, proposed, budget, weights);

    // a name org.json escapes: the host emitter, the same text as newAssignmentJson of planWaves
    std::vector<TopicInput> odd = topics;
    std::vector<TopicOutput> oddProposed = proposed;
    odd[5].name = oddProposed[5].name = "a\"b</c\\d";
    compare(a, odd, oddProposed, 2, {});
    const KafkaTopicAssigner::WaveDocs escaped = a.planWavesJson(odd, oddProposed, 1000000);
    CHECK(escaped.docs.size() == 1 && escaped.docs[0].find("\"a\\\"b<\\/c\\\\d\"") != std::string::npos);

    // argv[1]: a file of names the device refuses, one per line as "<hex of the name's UTF-8> <hex of its org.json quote>": each
    // takes the host emitter, and every record of its topic prints that quote
    if (argc > 1) {
        std::ifstream in(argv[1]);
        std::string nameHex, quoteHex;
        int n = 0;
        while (in >> nameHex >> quoteHex) {
            odd[5].name = oddProposed[5].name = unhex(nameHex);
            CHECK(kassign::needsJsonEscape(odd[5].name));
            compare(a, odd, oddProposed, 2, {});
            const KafkaTopicAssigner::WaveDocs one = a.planWavesJson(odd, oddProposed, 1000000);
            const std::string rec = ",\"topic\":" + unhex(quoteHex) + "}";
            size_t hits = 0;
            for (size_t at = one.docs.empty() ? std::string::npos : one.docs[0].find(rec); at != std::string::npos;
                 at = one.docs[0].find(rec, at + 1))
                ++hits;
            size_t moved = 0;
            for (const auto& e : oddProposed[5].assignment) moved += e.second != odd[5].current.at(e.first);
            CHECK(one.status.code == KA_OK && one.docs.size() == 1 && moved > 0 && hits == moved);
            ++n;
        }
        CHECK(n > 0);
    }
    // a NUL in a name would cut its hash short: refused before anything runs
    std::vector<TopicInput> nul = topics;
    nul[3].name = std::string("t\0x", 3);
    bool threw = false;
    try { a.planWavesJson(nul, proposed, 2); } catch (const std::invalid_argument&) { threw = true; }
    CHECK(threw);

    // nothing changed: no document
    std::vector<TopicOutput> same;
    for (const TopicInput& t : topics) same.push_back(TopicOutput{t.name, t.current});
    const KafkaTopicAssigner::WaveDocs none = a.planWavesJson(topics, same, 1);
    CHECK(none.status.code == KA_OK && none.docs.empty() && none.summary.empty());

    // a proposal naming a broker twice is refused with its row and broker
    std::vector<TopicOutput> bad = proposed;
    bad[2].assignment.begin()->second = {7, 7};
    const KafkaTopicAssigner::WaveDocs refused = a.planWavesJson(topics, bad, 3);
    CHECK(refused.status.code == KA_ERR_BAD_ARG && refused.status.b == 7 && refused.docs.empty() && refused.summary.empty());
    CHECK(refused.status.a == (int)(topics[0].current.size() + topics[1].current.size()));
    if (failures) {
        std::printf("FAILED %d\n", failures);
        return 1;
    }
    std::printf("OK\n");
    return 0;
}
