// kafka_assignment_generator.cpp — file-based front end with the reference tool's flag surface and output format,
// driving the GPU solver through kassign_host.hpp. Mirrors siftscience.kafka.tools.KafkaAssignmentGenerator
// (reference KafkaAssignmentGenerator.java:48-304) with ONE substitution: the ZooKeeper reads (KAG:273-276 and the
// ZkUtils calls at KAG:106-110, 114, 140, 157, 163) are replaced by a cluster snapshot file, because the ZK/Kafka client
// stack is out of scope (SURVEY §8f row 1). Everything downstream of the reads — broker resolution, exclusion, rack
// filtering, topic order, the solve, and the printed JSON — follows the reference.
//
//   kafka-assignment-generator --zk_string file:/path/snapshot.json --mode PRINT_REASSIGNMENT
//        [--broker_hosts h1,h2 | --integer_broker_ids 1,2] [--broker_hosts_to_remove h3] [--topics a,b]
//        [--desired_replication_factor N] [--disable_rack_awareness]
//
// Snapshot JSON: {"brokers":[{"id":1,"host":"h1","port":9092,"rack":"a"}, ...],          (PRINT_CURRENT_BROKERS shape, KAG:113-129)
//                 "topics":["t1", ...],                                                    (order of ZkUtils.getAllTopics; optional)
//                 "partitions":[{"topic":"t1","partition":0,"replicas":[1,2]}, ...]}       (Kafka reassignment shape)
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <sstream>
#include <unordered_map>

#include "kassign_host.hpp"

namespace {

// ---- a minimal JSON reader (objects, arrays, strings, integers, true/false/null) -----------------------------------
struct JVal {
    enum Kind { Null, Bool, Num, Str, Arr, Obj } kind = Null;
    bool b = false;
    long long num = 0;
    std::string str;
    std::vector<JVal> arr;
    std::vector<std::pair<std::string, JVal>> obj;
    const JVal* get(const std::string& k) const {
        for (const auto& kv : obj)
            if (kv.first == k) return &kv.second;
        return nullptr;
    }
};

struct JParser {
    const std::string& s;
    size_t i = 0;
    explicit JParser(const std::string& src) : s(src) {}
    [[noreturn]] void fail(const char* what) { throw std::runtime_error(std::string("snapshot JSON: ") + what + " at byte " + std::to_string(i)); }
    void ws() { while (i < s.size() && (s[i] == ' ' || s[i] == '\n' || s[i] == '\t' || s[i] == '\r')) ++i; }
    // the four hex digits of a \u escape at i
    unsigned hex4() {
        if (i + 4 > s.size()) fail("bad \\u escape");
        const unsigned cp = (unsigned)std::stoul(s.substr(i, 4), nullptr, 16);
        i += 4;
        return cp;
    }
    JVal parse() {
        ws();
        if (i >= s.size()) fail("unexpected end");
        JVal v;
        char c = s[i];
        if (c == '{') {
            v.kind = JVal::Obj;
            ++i; ws();
            if (i < s.size() && s[i] == '}') { ++i; return v; }
            for (;;) {
                ws();
                JVal k = parse();
                if (k.kind != JVal::Str) fail("object key must be a string");
                ws();
                if (i >= s.size() || s[i] != ':') fail("expected ':'");
                ++i;
                v.obj.emplace_back(k.str, parse());
                ws();
                if (i < s.size() && s[i] == ',') { ++i; continue; }
                if (i < s.size() && s[i] == '}') { ++i; break; }
                fail("expected ',' or '}'");
            }
        } else if (c == '[') {
            v.kind = JVal::Arr;
            ++i; ws();
            if (i < s.size() && s[i] == ']') { ++i; return v; }
            for (;;) {
                v.arr.push_back(parse());
                ws();
                if (i < s.size() && s[i] == ',') { ++i; continue; }
                if (i < s.size() && s[i] == ']') { ++i; break; }
                fail("expected ',' or ']'");
            }
        } else if (c == '"') {
            v.kind = JVal::Str;
            ++i;
            while (i < s.size() && s[i] != '"') {
                if (s[i] == '\\' && i + 1 < s.size()) {
                    char e = s[i + 1];
                    i += 2;
                    switch (e) {
                    case 'n': v.str.push_back('\n'); break;
                    case 't': v.str.push_back('\t'); break;
                    case 'r': v.str.push_back('\r'); break;
                    case 'b': v.str.push_back('\b'); break;
                    case 'f': v.str.push_back('\f'); break;
                    case 'u': {
                        unsigned cp = hex4();
                        // a high surrogate followed by a low one is one character (json.dumps writes every character above
                        // U+FFFF so); a lone surrogate keeps its own 3-byte form, which ka_java_string_hash reads as that unit
                        if (cp >= 0xD800 && cp < 0xDC00 && s.compare(i, 2, "\\u") == 0) {
                            const size_t at = i;
                            i += 2;
                            const unsigned lo = hex4();
                            if (lo >= 0xDC00 && lo < 0xE000) cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
                            else i = at;
                        }
                        if (cp < 0x80) v.str.push_back((char)cp);
                        else if (cp < 0x800) { v.str.push_back((char)(0xC0 | (cp >> 6))); v.str.push_back((char)(0x80 | (cp & 0x3F))); }
                        else if (cp < 0x10000) { v.str.push_back((char)(0xE0 | (cp >> 12))); v.str.push_back((char)(0x80 | ((cp >> 6) & 0x3F))); v.str.push_back((char)(0x80 | (cp & 0x3F))); }
                        else {
                            v.str.push_back((char)(0xF0 | (cp >> 18)));
                            v.str.push_back((char)(0x80 | ((cp >> 12) & 0x3F)));
                            v.str.push_back((char)(0x80 | ((cp >> 6) & 0x3F)));
                            v.str.push_back((char)(0x80 | (cp & 0x3F)));
                        }
                        break;
                    }
                    default: v.str.push_back(e);
                    }
                } else {
                    v.str.push_back(s[i++]);
                }
            }
            if (i >= s.size()) fail("unterminated string");
            ++i;
        } else if (c == '-' || (c >= '0' && c <= '9')) {
            v.kind = JVal::Num;
            size_t j = i;
            if (s[j] == '-') ++j;
            while (j < s.size() && s[j] >= '0' && s[j] <= '9') ++j;
            v.num = std::stoll(s.substr(i, j - i));
            i = j;
        } else if (s.compare(i, 4, "true") == 0) { v.kind = JVal::Bool; v.b = true; i += 4; }
        else if (s.compare(i, 5, "false") == 0) { v.kind = JVal::Bool; v.b = false; i += 5; }
        else if (s.compare(i, 4, "null") == 0) { v.kind = JVal::Null; i += 4; }
        else fail("unexpected character");
        return v;
    }
};

// ---- the cluster snapshot (what the reference reads from ZooKeeper) ---------------------------------------------------
struct Broker {
    int id;
    std::string host;
    int port;
    bool hasRack;
    std::string rack;
};

struct Snapshot {
    std::vector<Broker> brokers;                                    // ZkUtils.getAllBrokersInCluster
    std::vector<std::string> topics;                                // ZkUtils.getAllTopics (order preserved)
    std::unordered_map<std::string, kassign::Assignment> assignment;  // getPartitionAssignmentForTopics
};

Snapshot loadSnapshot(const std::string& path) {
    std::ifstream in(path, std::ios::binary);
    if (!in) throw std::runtime_error("cannot open cluster snapshot " + path);
    std::stringstream ss;
    ss << in.rdbuf();
    const std::string text = ss.str();
    JVal root = JParser(text).parse();
    Snapshot sn;
    // String.hashCode of a topic is taken over a C string: a name with a NUL would be solved with the hash of its prefix
    auto topicName = [](const JVal& t) -> const std::string& {
        if (t.str.find('\0') != std::string::npos) throw std::runtime_error("snapshot JSON: a topic name holds \\u0000");
        return t.str;
    };
    if (const JVal* bs = root.get("brokers"))
        for (const JVal& b : bs->arr) {
            Broker br{};
            const JVal* id = b.get("id");
            if (!id) throw std::runtime_error("snapshot broker without id");
            br.id = (int)id->num;
            if (const JVal* h = b.get("host")) br.host = h->str;
            if (const JVal* p = b.get("port")) br.port = (int)p->num;
            const JVal* r = b.get("rack");
            br.hasRack = r && r->kind == JVal::Str;
            if (br.hasRack) br.rack = r->str;
            sn.brokers.push_back(br);
        }
    if (const JVal* ps = root.get("partitions"))
        for (const JVal& p : ps->arr) {
            const JVal *t = p.get("topic"), *pi = p.get("partition"), *rs = p.get("replicas");
            if (!t || !pi || !rs) throw std::runtime_error("snapshot partition record needs topic/partition/replicas");
            auto& asg = sn.assignment[topicName(*t)];
            if (sn.assignment.size() > sn.topics.size() && !root.get("topics")) sn.topics.push_back(t->str);  // first-seen order
            std::vector<int>& reps = asg[(int)pi->num];
            reps.clear();
            for (const JVal& r : rs->arr) reps.push_back((int)r.num);
        }
    if (const JVal* ts = root.get("topics")) {
        sn.topics.clear();
        for (const JVal& t : ts->arr) sn.topics.push_back(topicName(t));
    }
    return sn;
}

// ---- option parsing (args4j @Option fields of KAG:53-84) -------------------------------------------------------------
struct Options {
    bool haveZk = false, haveMode = false;
    std::string zkConnectString, mode;
    bool haveBrokerIds = false, haveBrokerHosts = false, haveRemove = false, haveTopics = false;
    std::string brokerIds, brokerHostnames, brokerHostnamesToReplace, topics;
    int desiredReplicationFactor = -1;
    bool disableRackAwareness = false;
};

void printUsage() {
    // KAG:267-268: script line + args4j usage, to stderr
    std::fprintf(stderr,
                 "./kafka-assignment-generator.sh [options...] arguments...\n"
                 " --broker_hosts VAL                     : comma-separated list of broker\n"
                 "                                          hostnames (instead of broker IDs)\n"
                 " --broker_hosts_to_remove VAL           : comma-separated list of broker\n"
                 "                                          hostnames to exclude (instead of\n"
                 "                                          broker IDs)\n"
                 " --desired_replication_factor N         : used for changing replication factor\n"
                 "                                          for topics, if not present it will use\n"
                 "                                          the existing number\n"
                 " --disable_rack_awareness               : set to true to ignore rack\n"
                 "                                          configurations\n"
                 " --integer_broker_ids VAL               : comma-separated list of Kafka broker\n"
                 "                                          IDs (integers)\n"
                 " --mode [PRINT_CURRENT_ASSIGNMENT |     : the mode to run (PRINT_CURRENT_ASSIGNM\n"
                 " PRINT_CURRENT_BROKERS |                  ENT, PRINT_CURRENT_BROKERS,\n"
                 " PRINT_REASSIGNMENT]                      PRINT_REASSIGNMENT)\n"
                 " --topics VAL                           : comma-separated list of topics\n"
                 " --zk_string VAL                        : ZK quorum as comma-separated\n"
                 "                                          host:port pairs (here: file:<cluster\n"
                 "                                          snapshot json>)\n");
}

std::vector<std::string> splitComma(const std::string& s) {  // Guava Splitter.on(',') — keeps empty pieces
    std::vector<std::string> out;
    size_t a = 0;
    for (;;) {
        size_t b = s.find(',', a);
        out.push_back(s.substr(a, b == std::string::npos ? std::string::npos : b - a));
        if (b == std::string::npos) break;
        a = b + 1;
    }
    return out;
}

bool parseArgs(int argc, char** argv, Options& o) {
    for (int i = 1; i < argc; ++i) {
        const std::string a = argv[i];
        auto val = [&](std::string& dst, bool& have) {
            if (i + 1 >= argc) return false;  // args4j: "Option ... takes an operand"
            dst = argv[++i];
            have = true;
            return true;
        };
        bool dummy = false;
        if (a == "--zk_string") { if (!val(o.zkConnectString, o.haveZk)) return false; }
        else if (a == "--mode") { if (!val(o.mode, o.haveMode)) return false; }
        else if (a == "--integer_broker_ids") { if (!val(o.brokerIds, o.haveBrokerIds)) return false; }
        else if (a == "--broker_hosts") { if (!val(o.brokerHostnames, o.haveBrokerHosts)) return false; }
        else if (a == "--broker_hosts_to_remove") { if (!val(o.brokerHostnamesToReplace, o.haveRemove)) return false; }
        else if (a == "--topics") { if (!val(o.topics, o.haveTopics)) return false; }
        else if (a == "--desired_replication_factor") {
            std::string v;
            if (!val(v, dummy)) return false;
            char* end = nullptr;
            long n = std::strtol(v.c_str(), &end, 10);
            if (end == v.c_str() || *end) return false;  // args4j: not a valid int
            o.desiredReplicationFactor = (int)n;
        } else if (a == "--disable_rack_awareness") { o.disableRackAwareness = true; }
        else return false;  // unknown option / stray argument -> CmdLineException
    }
    if (!o.haveZk || !o.haveMode) return false;                                   // checkNotNull KAG:260-261
    if (o.mode != "PRINT_CURRENT_ASSIGNMENT" && o.mode != "PRINT_CURRENT_BROKERS" && o.mode != "PRINT_REASSIGNMENT") return false;
    if (o.haveBrokerIds && o.haveBrokerHosts) return false;                       // checkArgument KAG:262-264
    return true;
}

// KAG:189-204
std::set<int> brokerHostnamesToBrokerIds(const Snapshot& sn, const std::set<std::string>& hosts, bool checkPresence) {
    std::set<int> ids;
    for (const Broker& b : sn.brokers)
        if (hosts.count(b.host)) ids.insert(b.id);
    if (checkPresence && hosts.size() != ids.size()) {
        std::string found = "[";
        bool first = true;
        for (int id : ids) { if (!first) found += ", "; first = false; found += std::to_string(id); }
        throw std::invalid_argument("Some hostnames could not be found! We found: " + found + "]");
    }
    return ids;
}

std::string currentBrokersJson(const Snapshot& sn) {
    // org.json key order == HashMap bucket order of the keys (predicted, see kassign_host.hpp): rack, port, host, id
    std::string s = "[";
    for (size_t i = 0; i < sn.brokers.size(); ++i) {
        const Broker& b = sn.brokers[i];
        if (i) s.push_back(',');
        s.push_back('{');
        if (b.hasRack) { s += "\"rack\":"; kassign::appendQuoted(s, b.rack); s.push_back(','); }
        s += "\"port\":"; kassign::appendInt(s, b.port);
        s += ",\"host\":"; kassign::appendQuoted(s, b.host);
        s += ",\"id\":"; kassign::appendInt(s, b.id);
        s.push_back('}');
    }
    s.push_back(']');
    return s;
}

std::vector<kassign::TopicInput> gatherTopics(const Snapshot& sn, const std::vector<std::string>& names, bool failIfMissing) {
    std::vector<kassign::TopicInput> out;
    for (const std::string& n : names) {
        auto it = sn.assignment.find(n);
        if (it == sn.assignment.end()) {
            // ZkUtils.getPartitionAssignmentForTopics yields an EMPTY map for a topic without partition records, so
            // generateAssignment sees zero partitions: "Topic X does not have a positive replication factor!" (KTA:65-66), or
            // no rows at all with --desired_replication_factor > 0. The solver reproduces both from an empty Assignment.
            if (failIfMissing) out.push_back({n, kassign::Assignment{}});
            continue;
        }
        out.push_back({n, it->second});
    }
    return out;
}

int runTool(int argc, char** argv) {
    Options o;
    if (!parseArgs(argc, argv, o)) {  // KAG:258-270: any parse/validation failure -> usage on stderr, normal return
        printUsage();
        return 0;
    }
    std::string path = o.zkConnectString;
    if (path.rfind("file:", 0) == 0) path = path.substr(5);
    Snapshot sn = loadSnapshot(path);

    // getTopics KAG:252-254
    const bool topicsSpecified = o.haveTopics;
    std::vector<std::string> topics = topicsSpecified ? splitComma(o.topics) : sn.topics;

    // getBrokerIds KAG:206-225
    std::set<int> brokerIdSet;
    if (o.haveBrokerIds && !o.brokerIds.empty()) {
        for (const std::string& t : splitComma(o.brokerIds)) {
            char* end = nullptr;
            long v = std::strtol(t.c_str(), &end, 10);
            if (t.empty() || *end) throw std::invalid_argument("Invalid broker ID: " + t);
            brokerIdSet.insert((int)v);
        }
    } else if (o.haveBrokerHosts && !o.brokerHostnames.empty()) {
        auto hs = splitComma(o.brokerHostnames);
        brokerIdSet = brokerHostnamesToBrokerIds(sn, std::set<std::string>(hs.begin(), hs.end()), true);
    }
    // getExcludedBrokerIds KAG:227-236
    std::set<int> excluded;
    if (o.haveRemove && !o.brokerHostnamesToReplace.empty()) {
        auto hs = splitComma(o.brokerHostnamesToReplace);
        excluded = brokerHostnamesToBrokerIds(sn, std::set<std::string>(hs.begin(), hs.end()), false);
    }
    // getRackAssignment KAG:238-250
    std::map<int, std::string> rackAssignment;
    if (!o.disableRackAwareness)
        for (const Broker& b : sn.brokers)
            if (b.hasRack) rackAssignment[b.id] = b.rack;

    if (o.mode == "PRINT_CURRENT_ASSIGNMENT") {  // KAG:103-111
        std::cout << "CURRENT ASSIGNMENT:\n" << kassign::kafkaReassignmentJson(gatherTopics(sn, topics, false)) << "\n";
    } else if (o.mode == "PRINT_CURRENT_BROKERS") {  // KAG:113-129
        std::cout << "CURRENT BROKERS:\n" << currentBrokersJson(sn) << "\n";
    } else {  // PRINT_REASSIGNMENT, KAG:131-187
        std::set<int> brokerSet = brokerIdSet;
        if (brokerSet.empty())
            for (const Broker& b : sn.brokers) brokerSet.insert(b.id);           // KAG:137-147
        std::set<int> brokers;
        for (int b : brokerSet)
            if (!excluded.count(b)) brokers.insert(b);                           // Sets.difference KAG:150
        for (auto it = rackAssignment.begin(); it != rackAssignment.end();)      // retainAll KAG:151
            it = brokers.count(it->first) ? std::next(it) : rackAssignment.erase(it);
        std::cout << "CURRENT ASSIGNMENT:\n" << kassign::kafkaReassignmentJson(gatherTopics(sn, topics, false)) << "\n";  // KAG:160
        std::vector<kassign::TopicInput> inputs = gatherTopics(sn, topics, true);
        kassign::KafkaTopicAssigner assigner;                                   // ONE assigner for the run, KAG:172
        const std::string result = assigner.solveTopicsJson(inputs, brokers, rackAssignment, o.desiredReplicationFactor);
        std::cout << "NEW ASSIGNMENT:\n" << result << "\n";                    // KAG:186, text built on the device
    }
    return 0;
}

}  // namespace

int main(int argc, char** argv) {
    try {
        return runTool(argc, argv);
    } catch (const kassign::IllegalStateException& e) {
        std::fprintf(stderr, "Exception in thread \"main\" java.lang.IllegalStateException: %s\n", e.what());
    } catch (const kassign::ArrayIndexOutOfBoundsException& e) {
        std::fprintf(stderr, "Exception in thread \"main\" java.lang.ArrayIndexOutOfBoundsException: %s\n", e.what());
    } catch (const std::invalid_argument& e) {
        std::fprintf(stderr, "Exception in thread \"main\" java.lang.IllegalArgumentException: %s\n", e.what());
    } catch (const std::exception& e) {
        std::fprintf(stderr, "Exception in thread \"main\" %s\n", e.what());
    }
    return 1;  // uncaught exception in the reference: stack trace + non-zero exit, no NEW ASSIGNMENT printed
}
