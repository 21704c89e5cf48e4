// test_candidate_scores.cpp — KafkaTopicAssigner::scoreTopicsCandidates against the summary computed here from the assignments
// solveTopicsCandidates returns: per candidate the rows changed / moved, leaders changed, replicas added / dropped (weighted),
// the per-broker sums and their extremes; failed candidates are zero and carry the exception solveTopicsCandidates reports.
// Needs a GPU (kassign has no CPU fallback). Exit code 0 = all passed.
#include <algorithm>
#include <climits>
#include <cstdio>
#include <cstdlib>

#include "kassign_host.hpp"

using kassign::KafkaTopicAssigner;
using kassign::TopicInput;

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

static KafkaTopicAssigner::Candidate candidate(int lo, int hi, int racks) {
    KafkaTopicAssigner::Candidate c;
    for (int b = lo; b <= hi; ++b) {
        c.brokers.insert(b);
        if (racks > 0) c.rackAssignment[b] = "rack" + std::to_string(b % racks);
    }
    return c;
}

// The summary of one candidate's assignment against the current one, by the definitions of ka_move_summary.
static KafkaTopicAssigner::CandidateScore expected(const std::vector<TopicInput>& topics, const KafkaTopicAssigner::CandidateResult& r,
                                                   const KafkaTopicAssigner::Candidate& c, const std::vector<std::map<int, int64_t>>& w) {
    KafkaTopicAssigner::CandidateScore e{};
    e.summary.max_broker_in_id = -1;
    for (int b : c.brokers) e.brokerReplicas[b] = e.brokerLeaders[b] = e.brokerIn[b] = 0;
    ka_move_summary& s = e.summary;
    for (size_t t = 0; t < topics.size(); ++t)
        for (const auto& p : topics[t].current) {
            const std::vector<int>& cur = p.second;
            const std::vector<int>& nw = r.topics[t].assignment.at(p.first);
            const int64_t wt = w.empty() ? 1 : w[t].at(p.first);
            auto has = [](const std::vector<int>& v, int b) { return std::find(v.begin(), v.end(), b) != v.end(); };
            int64_t add = 0, drop = 0;
            for (int b : nw) {
                e.brokerReplicas[b] += wt;
                if (!has(cur, b)) { ++add; e.brokerIn[b] += wt; }
            }
            for (int b : cur) drop += !has(nw, b);
            if (!nw.empty()) e.brokerLeaders[nw[0]] += wt;
            s.rows_changed += nw != cur;
            s.rows_moved += add + drop > 0;
            s.leaders_changed += cur.empty() || nw.empty() || nw[0] != cur[0];
            s.replicas_added += wt * add;
            s.replicas_dropped += wt * drop;
        }
    s.min_broker_replicas = s.min_broker_leaders = LLONG_MAX;
    for (int b : c.brokers) {   // ascending: the first maximum is the lowest id
        if (e.brokerIn[b] > s.max_broker_in) { s.max_broker_in = e.brokerIn[b]; s.max_broker_in_id = b; }
        s.max_broker_replicas = std::max<int64_t>(s.max_broker_replicas, e.brokerReplicas[b]);
        s.min_broker_replicas = std::min<int64_t>(s.min_broker_replicas, e.brokerReplicas[b]);
        s.max_broker_leaders = std::max<int64_t>(s.max_broker_leaders, e.brokerLeaders[b]);
        s.min_broker_leaders = std::min<int64_t>(s.min_broker_leaders, e.brokerLeaders[b]);
    }
    return e;
}

static bool sameSummary(const ka_move_summary& a, const ka_move_summary& b) {
    return a.rows_changed == b.rows_changed && a.rows_moved == b.rows_moved && a.leaders_changed == b.leaders_changed &&
           a.replicas_added == b.replicas_added && a.replicas_dropped == b.replicas_dropped && a.max_broker_in == b.max_broker_in &&
           a.max_broker_in_id == b.max_broker_in_id && a.max_broker_replicas == b.max_broker_replicas &&
           a.min_broker_replicas == b.min_broker_replicas && a.max_broker_leaders == b.max_broker_leaders &&
           a.min_broker_leaders == b.min_broker_leaders;
}

static void testScoresMatchTheAssignments() {
    const std::vector<TopicInput> topics = makeTopics(11u, 60, 30, 12);   // 3 or 4 of the first four candidates solve
    const std::vector<KafkaTopicAssigner::Candidate> cands = {
        candidate(1, 30, 0), candidate(1, 24, 0), candidate(1, 30, 4), candidate(3, 40, 5),
        candidate(1, 2, 0),     // fewer brokers than RF 3
        candidate(1, 0, 0),     // no broker at all
    };
    std::vector<std::map<int, int64_t>> weights(topics.size());
    unsigned seed = 5u;
    for (size_t t = 0; t < topics.size(); ++t)
        for (const auto& p : topics[t].current) { seed = seed * 1103515245u + 12345u; weights[t][p.first] = (int64_t)(seed >> 4) << 12; }
    KafkaTopicAssigner a;
    for (int desired : {-1, 2, 3}) {
        const auto rows = a.solveTopicsCandidates(topics, cands, desired);
        const std::vector<std::map<int, int64_t>> none;
        for (bool weighted : {true, false}) {
            const auto& wt = weighted ? weights : none;
            const auto res = a.scoreTopicsCandidates(topics, cands, desired, wt, true);
            CHECK(res.size() == cands.size());
            int solved = 0;
            for (size_t k = 0; k < cands.size(); ++k) {
                CHECK(res[k].status.code == rows[k].status.code && res[k].status.topic_index == rows[k].status.topic_index &&
                      res[k].status.partition == rows[k].status.partition);
                if (rows[k].status.code != KA_OK) {
                    ka_move_summary zero{};
                    zero.max_broker_in_id = -1;
                    CHECK(sameSummary(res[k].summary, zero));
                    for (const auto& e : res[k].brokerReplicas) CHECK(e.second == 0);
                    continue;
                }
                ++solved;
                const auto e = expected(topics, rows[k], cands[k], wt);
                if (!sameSummary(res[k].summary, e.summary)) {
                    std::fprintf(stderr, "candidate %zu desired %d: summaries differ\n", k, desired);
                    ++failures;
                }
                CHECK(res[k].brokerReplicas == e.brokerReplicas && res[k].brokerLeaders == e.brokerLeaders && res[k].brokerIn == e.brokerIn);
            }
            CHECK(solved >= 3);
        }
    }
    // a failing candidate reports the exception solveTopicsCandidates reports
    const auto res = a.scoreTopicsCandidates(topics, {candidate(1, 2, 0)}, -1);
    std::vector<std::string> names;
    for (const auto& t : topics) names.push_back(t.name);
    try { kassign::throwForStatus(res[0].status, names); CHECK(false); }
    catch (const kassign::IllegalStateException& e) { CHECK(std::string(e.what()).find("higher replication factor") != std::string::npos); }
}

int main() {
    try {
        testScoresMatchTheAssignments();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 2;
    }
    std::printf("%s (%d failure%s)\n", failures ? "FAILED" : "OK", failures, failures == 1 ? "" : "s");
    return failures ? 1 : 0;
}
