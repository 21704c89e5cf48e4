// test_broker_usage.cpp — KafkaTopicAssigner::brokerUsage over a planWaves plan of the rows of solveTopics with a drained broker:
// every field equals a plain loop over the waves of the rule of include/kassign.h; the same plan run as one wave peaks at what
// each broker holds before plus what it receives; a receiver missing from the usage table is refused with its row and id.
// With a file argument the test also writes the flat inputs and the report there, for the Python side to compare
// Solver.broker_usage with. Needs a GPU (kassign has no CPU fallback). Exit code 0 = all passed.
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

// One partition of the flat row order: its current and new list, weight and wave.
struct Row {
    std::vector<int> cur, next;
    int64_t w;
    int wave;
};

// The rule, one wave at a time: before, usage(v) for v = 0..W, peak, after, over.
static ka_broker_usage model(const std::vector<Row>& rows, int b, int64_t base, int64_t cap, bool capped, int W) {
    auto has = [](const std::vector<int>& l, int x) { return std::find(l.begin(), l.end(), x) != l.end(); };
    int64_t before = base;
    for (const Row& r : rows) before += has(r.cur, b) ? r.w : 0;
    ka_broker_usage u{before, before, 0, 0, capped && before > cap ? 0 : -1};
    int64_t last = before;
    for (int v = 0; v <= W; ++v) {
        int64_t x = before;
        for (const Row& r : rows) {
            if (r.wave >= 1 && r.wave <= v && has(r.next, b) && !has(r.cur, b)) x += r.w;
            if (r.wave >= 1 && r.wave < v && has(r.cur, b) && !has(r.next, b)) x -= r.w;
        }
        if (x > u.peak) { u.peak = x; u.peak_wave = v; }
        if (u.over_wave < 0 && capped && x > cap) u.over_wave = v;
        last = x;
    }
    for (const Row& r : rows)
        if (W >= 1 && r.wave == W && has(r.cur, b) && !has(r.next, b)) last -= r.w;
    u.after = last;
    return u;
}

int main(int argc, char** argv) {
    KafkaTopicAssigner a(0);
    const int nb = 24;
    const std::vector<TopicInput> topics = makeTopics(77, 60, nb, 40);
    std::set<int> brokers;
    for (int b = 2; b <= nb + 3; ++b) brokers.insert(b);   // broker 1 drained, brokers nb + 1 .. nb + 3 joined empty
    const std::vector<TopicOutput> proposed = a.solveTopics(topics, brokers, {}, -1);
    std::vector<std::map<int, int64_t>> weights(topics.size());
    for (size_t t = 0; t < topics.size(); ++t)
        for (const auto& e : topics[t].current) weights[t][e.first] = 1 + (int64_t)((t * 131 + e.first * 17) % 50);
    const KafkaTopicAssigner::WavePlan plan = a.planWaves(topics, proposed, 60, weights);
    CHECK(plan.status.code == KA_OK && plan.waves.size() > 2);
    std::vector<int32_t> ids;
    std::vector<int64_t> base, cap;
    for (int b = 1; b <= nb + 3; ++b) {
        ids.push_back(b);
        base.push_back(100 * (b % 7));
        cap.push_back(900 + 25 * (b % 5));
    }
    // the flat rows and their waves, as brokerUsage hands them over
    std::map<std::pair<std::string, int>, int> waveOf;
    for (size_t v = 0; v < plan.waves.size(); ++v)
        for (const TopicOutput& t : plan.waves[v])
            for (const auto& e : t.assignment) waveOf[{t.name, e.first}] = (int)v + 1;
    std::vector<Row> rows;
    for (size_t t = 0; t < topics.size(); ++t)
        for (const auto& e : topics[t].current) {
            const auto it = waveOf.find({topics[t].name, e.first});
            rows.push_back(Row{e.second, proposed[t].assignment.at(e.first), weights[t].at(e.first), it == waveOf.end() ? 0 : it->second});
        }
    const int W = (int)plan.waves.size();

    const KafkaTopicAssigner::BrokerUsage u = a.brokerUsage(topics, proposed, plan, ids, base, cap, weights);
    CHECK(u.status.code == KA_OK && u.waves == W && u.usage.size() == ids.size());
    int inside = 0;   // brokers whose peak lies strictly above both ends
    for (size_t i = 0; i < ids.size() && u.status.code == KA_OK; ++i) {
        const ka_broker_usage e = model(rows, ids[i], base[i], cap[i], true, W);
        const ka_broker_usage& g = u.usage.at(ids[i]);
        CHECK(g.before == e.before && g.peak == e.peak && g.peak_wave == e.peak_wave && g.after == e.after && g.over_wave == e.over_wave);
        inside += g.peak > std::max(g.before, g.after);
    }
    CHECK(u.usage.at(1).after == base[0]);   // the drained broker ends with its base alone
    std::printf("brokers with a peak above both ends: %d\n", inside);

    // the whole plan as one wave: the peak is before + what the broker receives
    KafkaTopicAssigner::WavePlan one = plan;
    one.waves.assign(1, {});
    for (const auto& w : plan.waves) one.waves[0].insert(one.waves[0].end(), w.begin(), w.end());
    const KafkaTopicAssigner::BrokerUsage u1 = a.brokerUsage(topics, proposed, one, ids, {}, {}, weights);
    CHECK(u1.status.code == KA_OK && u1.waves == 1);
    for (int32_t b : ids) {
        int64_t in = 0;
        for (const Row& r : rows)
            if (r.wave > 0 && std::find(r.next.begin(), r.next.end(), b) != r.next.end() &&
                std::find(r.cur.begin(), r.cur.end(), b) == r.cur.end())
                in += r.w;
        const ka_broker_usage& g = u1.usage.at(b);
        CHECK(g.peak == g.before + in && g.over_wave == -1);
    }

    // a receiver the usage table lacks: the lowest such row, with its id
    const std::vector<int32_t> without(ids.begin(), ids.end() - 1);
    const KafkaTopicAssigner::BrokerUsage bad = a.brokerUsage(topics, proposed, plan, without, {}, {}, weights);
    CHECK(bad.status.code == KA_ERR_BAD_ARG && bad.status.b == nb + 3 && bad.usage.empty());
    if (bad.status.code == KA_ERR_BAD_ARG) {
        const Row& r = rows.at(bad.status.a);
        CHECK(r.wave > 0 && std::find(r.next.begin(), r.next.end(), nb + 3) != r.next.end());
        for (int g = 0; g < bad.status.a; ++g)
            CHECK(rows[g].wave == 0 || std::find(rows[g].next.begin(), rows[g].next.end(), nb + 3) == rows[g].next.end() ||
                  std::find(rows[g].cur.begin(), rows[g].cur.end(), nb + 3) != rows[g].cur.end());
    }

    if (argc > 1 && u.status.code == KA_OK) {   // the flat inputs and the report, one array per line
        FILE* fp = std::fopen(argv[1], "w");
        CHECK(fp != nullptr);
        if (fp) {
            size_t stride = 1;
            for (const Row& r : rows) stride = std::max(stride, r.next.size());
            std::fprintf(fp, "%zu %zu %zu %d\n", rows.size(), stride, ids.size(), u.waves);
            auto line = [&](auto each) { each(); std::fprintf(fp, "\n"); };
            int64_t off = 0;
            line([&] { std::fprintf(fp, "0"); for (const Row& r : rows) std::fprintf(fp, " %lld", (long long)(off += r.cur.size())); });
            line([&] { for (const Row& r : rows) for (int b : r.cur) std::fprintf(fp, "%d ", b); });
            line([&] { for (const Row& r : rows) std::fprintf(fp, "%zu ", r.next.size()); });
            line([&] { for (const Row& r : rows) for (size_t j = 0; j < stride; ++j) std::fprintf(fp, "%d ", j < r.next.size() ? r.next[j] : -1); });
            line([&] { for (const Row& r : rows) std::fprintf(fp, "%lld ", (long long)r.w); });
            line([&] { for (const Row& r : rows) std::fprintf(fp, "%d ", r.wave); });
            line([&] { for (int32_t b : ids) std::fprintf(fp, "%d ", b); });
            line([&] { for (int64_t x : base) std::fprintf(fp, "%lld ", (long long)x); });
            line([&] { for (int64_t x : cap) std::fprintf(fp, "%lld ", (long long)x); });
            line([&] {
                for (int32_t b : ids) {
                    const ka_broker_usage& g = u.usage.at(b);
                    std::fprintf(fp, "%lld %lld %lld %lld %lld ", (long long)g.before, (long long)g.peak, (long long)g.peak_wave,
                                 (long long)g.after, (long long)g.over_wave);
                }
            });
            std::fclose(fp);
        }
    }
    if (failures) {
        std::fprintf(stderr, "%d failures\n", failures);
        return 1;
    }
    std::printf("OK\n");
    return 0;
}
