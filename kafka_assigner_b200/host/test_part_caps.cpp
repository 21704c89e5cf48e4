// test_part_caps.cpp — KafkaTopicAssigner::setPartCaps over the rows of solveTopics: the caps read back, a negative cap throws
// and leaves them; under a row cap every part holds at most that many partitions and joined in order the parts of every wave
// are still that wave's planWavesJson document; a row cap of 1 gives one part per changed partition; the plan and its
// summaries are those of the uncapped call; names that org.json escapes take the host cut, which cuts like the device; caps
// cleared to 0 give the uncapped parts again. Needs a GPU (kassign has no CPU fallback). Exit code 0 = all passed.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "kassign_host.hpp"

using kassign::KafkaTopicAssigner;
using kassign::TopicInput;
using kassign::TopicOutput;
using Caps = std::pair<int64_t, int64_t>;

static int failures = 0;
#define CHECK(cond)                                                              \
    do {                                                                         \
        if (!(cond)) { std::fprintf(stderr, "FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); ++failures; } \
    } while (0)

static const std::string kHead = "{\"partitions\":[", kTail = "],\"version\":1}";

// The seeded ragged run of test_waves_json.cpp.
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

// The records of a document, each without its comma (the names here hold no '}' or ',' inside a record's end).
static std::vector<std::string> records(const std::string& doc) {
    std::vector<std::string> out;
    const std::string body = doc.substr(kHead.size(), doc.size() - kHead.size() - kTail.size());
    size_t at = 0;
    while (at < body.size()) {
        const size_t end = body.find("},{", at);
        const size_t stop = end == std::string::npos ? body.size() : end + 1;
        out.push_back(body.substr(at, stop - at));
        at = stop + 1;
    }
    return out;
}

// How many records every part holds, and the wave of every part.
static std::vector<std::pair<size_t, int32_t>> shape(const KafkaTopicAssigner::WaveParts& p) {
    std::vector<std::pair<size_t, int32_t>> out;
    for (size_t d = 0; d < p.parts.size(); ++d) out.emplace_back(records(p.parts[d]).size(), p.partWave[d]);
    return out;
}

int main() {
    std::vector<TopicInput> topics = makeTopics(11, 300, 30, 12);
    std::set<int> brokers;
    std::map<int, std::string> racks;
    for (int b = 1; b <= 40; ++b) {   // brokers 31..40 joined empty
        brokers.insert(b);
        racks[b] = "rack" + std::to_string(b % 5);
    }
    KafkaTopicAssigner a;
    const std::vector<TopicOutput> proposed = a.solveTopics(topics, brokers, racks, -1);
    std::vector<std::map<int, int64_t>> weights(topics.size());
    unsigned seed = 5;
    for (size_t t = 0; t < topics.size(); ++t)
        for (const auto& p : topics[t].current) { seed = seed * 1103515245u + 12345u; weights[t][p.first] = (seed >> 8) % 100; }

    CHECK(a.partCaps() == Caps(0, 0));
    a.setPartCaps(7, 0);
    CHECK(a.partCaps() == Caps(7, 0));
    for (const Caps& bad : {Caps(-1, 0), Caps(0, -3)}) {
        bool threw = false;
        try {
            a.setPartCaps(bad.first, bad.second);
        } catch (const kassign::KassignError& e) {
            threw = e.code == KA_ERR_BAD_ARG;
        }
        CHECK(threw && a.partCaps() == Caps(7, 0));
    }
    a.setPartCaps(0, 0);

    const int64_t budget = 3;
    const KafkaTopicAssigner::WaveDocs docs = a.planWavesJson(topics, proposed, budget, weights);
    const KafkaTopicAssigner::WaveParts plain = a.planWaveParts(topics, proposed, budget, 4096, weights);
    CHECK(docs.status.code == KA_OK && plain.status.code == KA_OK);
    size_t changed = 0;
    for (const std::string& d : docs.docs) changed += records(d).size();

    // a row cap: at most Lr records a part, every wave's records in order, the plan of the uncapped call
    for (const int64_t rows : {1, 2, 5, 40}) {
        a.setPartCaps(rows, 0);
        const KafkaTopicAssigner::WaveParts parts = a.planWaveParts(topics, proposed, budget, 4096, weights);
        CHECK(parts.status.code == KA_OK && parts.summary.size() == docs.summary.size());
        CHECK(std::memcmp(parts.summary.data(), docs.summary.data(), docs.summary.size() * sizeof(ka_wave_summary)) == 0);
        size_t d = 0;
        for (size_t v = 0; v < docs.docs.size(); ++v) {
            std::vector<std::string> joined;
            for (; d < parts.parts.size() && parts.partWave[d] == (int32_t)v + 1; ++d) {
                const std::vector<std::string> r = records(parts.parts[d]);
                CHECK((int64_t)r.size() <= rows && (int64_t)parts.parts[d].size() <= 4096);
                joined.insert(joined.end(), r.begin(), r.end());
            }
            CHECK(joined == records(docs.docs[v]));
        }
        CHECK(d == parts.parts.size() && parts.parts.size() >= plain.parts.size());
        if (rows == 1) CHECK(parts.parts.size() == changed);
        const KafkaTopicAssigner::WaveRollback back = a.planWavePartsRollback(topics, proposed, budget, 1 << 20, weights);
        CHECK(back.status.code == KA_OK && back.parts.size() == back.rollback.size());
        for (const std::string& p : back.parts) CHECK((int64_t)records(p).size() <= rows);
    }

    // a name org.json escapes takes the host cut; with a limit that never binds, it cuts like the device under both caps
    std::vector<TopicInput> odd = topics;
    std::vector<TopicOutput> oddProposed = proposed;
    odd[5].name = oddProposed[5].name = "a\"b</c\\d";
    for (const Caps& caps : {Caps(3, 0), Caps(0, 1), Caps(0, 150), Caps(4, 200)}) {
        a.setPartCaps(caps.first, caps.second);
        for (const bool weighted : {true, false}) {
            const std::vector<std::map<int, int64_t>> wt = weighted ? weights : std::vector<std::map<int, int64_t>>{};
            const KafkaTopicAssigner::WaveParts device = a.planWaveParts(topics, proposed, budget, 1 << 30, wt);
            const KafkaTopicAssigner::WaveParts host = a.planWaveParts(odd, oddProposed, budget, 1 << 30, wt);
            CHECK(device.status.code == KA_OK && host.status.code == KA_OK);
            CHECK(shape(device) == shape(host));
            const KafkaTopicAssigner::WaveRollback hostBack = a.planWavePartsRollback(odd, oddProposed, budget, 1 << 30, wt);
            CHECK(hostBack.status.code == KA_OK && hostBack.parts == host.parts);
        }
    }

    // caps cleared: the uncapped parts again
    a.setPartCaps(0, 0);
    const KafkaTopicAssigner::WaveParts again = a.planWaveParts(topics, proposed, budget, 4096, weights);
    CHECK(again.status.code == KA_OK && again.parts == plain.parts && again.partWave == plain.partWave);
    if (failures) {
        std::printf("FAILED %d\n", failures);
        return 1;
    }
    std::printf("OK\n");
    return 0;
}
