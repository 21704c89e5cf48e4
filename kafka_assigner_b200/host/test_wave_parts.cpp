// test_wave_parts.cpp — KafkaTopicAssigner::planWaveParts over the rows of solveTopics: joined in order, the parts of every
// wave are that wave's planWavesJson document; every part is within the limit and could not take the next part's first
// record; a limit above every wave gives the documents of planWavesJson; names that org.json escapes take the host cut and
// give the same parts as the device would for their text; an over-long partition and a refused proposal carry their status.
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

static void compare(KafkaTopicAssigner& a, const std::vector<TopicInput>& topics, const std::vector<TopicOutput>& proposed,
                    int64_t budget, int64_t limit, const std::vector<std::map<int, int64_t>>& weights, const KafkaTopicAssigner::SendBudget* send) {
    const KafkaTopicAssigner::WaveDocs docs = send ? a.planWavesJson(topics, proposed, budget, *send, weights)
                                                   : a.planWavesJson(topics, proposed, budget, weights);
    const KafkaTopicAssigner::WaveParts parts = send ? a.planWaveParts(topics, proposed, budget, limit, *send, weights)
                                                     : a.planWaveParts(topics, proposed, budget, limit, weights);
    CHECK(docs.status.code == KA_OK && parts.status.code == KA_OK);
    CHECK(parts.summary.size() == docs.summary.size() && parts.parts.size() == parts.partWave.size());
    CHECK(std::memcmp(parts.summary.data(), docs.summary.data(), docs.summary.size() * sizeof(ka_wave_summary)) == 0);
    if (send) CHECK(std::memcmp(parts.sendSummary.data(), docs.sendSummary.data(), docs.sendSummary.size() * sizeof(ka_wave_send_summary)) == 0);
    size_t d = 0;
    for (size_t v = 0; v < docs.docs.size(); ++v) {
        std::vector<std::string> joined;
        for (size_t first = d; d < parts.parts.size() && parts.partWave[d] == (int32_t)v + 1; ++d) {
            CHECK((int64_t)parts.parts[d].size() <= limit);
            const std::vector<std::string> r = records(parts.parts[d]);
            if (d > first) CHECK((int64_t)(parts.parts[d - 1].size() + 1 + records(parts.parts[d]).front().size()) > limit);
            joined.insert(joined.end(), r.begin(), r.end());
        }
        CHECK(joined == records(docs.docs[v]));
    }
    CHECK(d == parts.parts.size());
}

int main() {
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
    KafkaTopicAssigner::SendBudget send{3, {}};
    for (int b = 1; b <= 40; ++b) send.sendBrokers.push_back(b);
    for (const int64_t limit : {100, 250, 4096, 1 << 20}) {
        for (const int64_t budget : {1, 4, 1000000}) compare(a, topics, proposed, budget, limit, {}, nullptr);
        compare(a, topics, proposed, 150, limit, weights, nullptr);
        compare(a, topics, proposed, 2, limit, {}, &send);
    }

    // a limit above every wave: the documents of planWavesJson, one part per wave
    const KafkaTopicAssigner::WaveDocs docs = a.planWavesJson(topics, proposed, 4);
    const KafkaTopicAssigner::WaveParts whole = a.planWaveParts(topics, proposed, 4, 1 << 30);
    CHECK(whole.parts == docs.docs && whole.partWave.size() == docs.docs.size());
    for (size_t v = 0; v < whole.partWave.size(); ++v) CHECK(whole.partWave[v] == (int32_t)v + 1);

    // a name org.json escapes: the host cut over the host emitter's records
    std::vector<TopicInput> odd = topics;
    std::vector<TopicOutput> oddProposed = proposed;
    odd[5].name = oddProposed[5].name = "a\"b</c\\d";
    for (const int64_t limit : {120, 1000, 1 << 20}) compare(a, odd, oddProposed, 2, limit, {}, nullptr);
    const KafkaTopicAssigner::WaveParts escaped = a.planWaveParts(odd, oddProposed, 1000000, 1 << 30);
    CHECK(escaped.parts.size() == 1 && escaped.parts[0].find("\"a\\\"b<\\/c\\\\d\"") != std::string::npos);

    // a partition whose one-record document exceeds the limit: its row and that length, on both paths
    for (const auto* in : {&topics, &odd}) {
        const std::vector<TopicOutput>& prop = in == &topics ? proposed : oddProposed;
        const KafkaTopicAssigner::WaveParts small = a.planWaveParts(*in, prop, 1000000, 40);
        CHECK(small.status.code == KA_ERR_LIMIT && small.status.b > 40 && small.parts.empty() && small.summary.empty());
    }

    // nothing changed: no part; a limit below 1 and a refused proposal carry their status
    std::vector<TopicOutput> same;
    for (const TopicInput& t : topics) same.push_back(TopicOutput{t.name, t.current});
    const KafkaTopicAssigner::WaveParts none = a.planWaveParts(topics, same, 1, 1000);
    CHECK(none.status.code == KA_OK && none.parts.empty() && none.partWave.empty() && none.summary.empty());
    CHECK(a.planWaveParts(topics, proposed, 1, 0).status.code == KA_ERR_BAD_ARG);
    std::vector<TopicOutput> bad = proposed;
    bad[2].assignment.begin()->second = {7, 7};
    const KafkaTopicAssigner::WaveParts refused = a.planWaveParts(topics, bad, 3, 1000);
    CHECK(refused.status.code == KA_ERR_BAD_ARG && refused.status.b == 7 && refused.parts.empty() && refused.summary.empty());
    if (failures) {
        std::printf("FAILED %d\n", failures);
        return 1;
    }
    std::printf("OK\n");
    return 0;
}
