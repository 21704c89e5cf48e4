"""The C++ host side: file-based kafka-assignment-generator with the reference tool's flags and output
(KafkaAssignmentGenerator.java:53-84, 103-187, 256-299). CPU tests cover flag handling and the two modes that need
no solve; the GPU test compares --mode PRINT_REASSIGNMENT byte-for-byte with JSON built from the oracle."""
import json
import os
import subprocess

import pytest

import kafka_assigner_b200 as kab
from oracle import py_oracle as po
from tests import models

BROKERS = [dict(id=10 + i, host="h%d" % (10 + i), port=9092, rack="abcd"[i % 4]) for i in range(8)] + [dict(id=18, host="h18", port=9093)]
TOPICS = {"test": {0: [10, 11], 1: [11, 12], 2: [12, 10], 3: [10, 12]},
          "events": {0: [13, 14, 10], 1: [14, 15, 11], 2: [15, 12, 13], 3: [10, 11, 12], 4: [12, 13, 14]},
          "logs.v2": {0: [11], 1: [12], 2: [15]}}
ORDER = ["events", "test", "logs.v2"]


@pytest.fixture(scope="module")
def cli(native_lib):
    return kab.build_mod.build_host()


@pytest.fixture()
def snapshot(tmp_path):
    parts = [dict(topic=t, partition=p, replicas=r) for t in ORDER for p, r in TOPICS[t].items()]
    path = tmp_path / "cluster.json"
    path.write_text(json.dumps(dict(brokers=BROKERS, topics=ORDER, partitions=parts)))
    return str(path)


def run(cli, *args):
    r = subprocess.run([cli] + list(args), capture_output=True, text=True, timeout=120)
    return r.returncode, r.stdout, r.stderr


def expected_new_assignment(topic_names, brokers, racks, desired=-1):
    recs = po.run_topics([(t, TOPICS[t]) for t in topic_names], brokers, racks, desired)
    return models.document(models.record(t, p, r) for t, p, r in recs)


def expected_current(topic_names):
    body = ",".join('{"topic":"%s","partition":%d,"replicas":[%s]}' % (t, p, ",".join(map(str, TOPICS[t][p])))
                    for t in topic_names for p in sorted(TOPICS[t]))
    return '{"version":1,"partitions":[' + body + ']}'


# ---- CPU ----------------------------------------------------------------------------------------------------------
def test_usage_on_missing_or_conflicting_flags(cli, snapshot):
    for args in ([], ["--mode", "PRINT_REASSIGNMENT"], ["--zk_string", snapshot], ["--zk_string", snapshot, "--mode", "NOPE"],
                 ["--zk_string", snapshot, "--mode", "PRINT_REASSIGNMENT", "--integer_broker_ids", "1", "--broker_hosts", "h10"],
                 ["--zk_string", snapshot, "--mode", "PRINT_REASSIGNMENT", "--bogus"],
                 ["--zk_string", snapshot, "--mode", "PRINT_REASSIGNMENT", "--desired_replication_factor", "x"]):
        rc, out, err = run(cli, *args)
        assert rc == 0 and out == ""                    # KAG:266-270: usage to stderr, plain return
        assert err.startswith("./kafka-assignment-generator.sh [options...] arguments...")
        assert "--broker_hosts_to_remove" in err and "--disable_rack_awareness" in err


def test_print_current_brokers_and_assignment(cli, snapshot):
    rc, out, _ = run(cli, "--zk_string", "file:" + snapshot, "--mode", "PRINT_CURRENT_BROKERS")
    assert rc == 0
    head, body = out.strip().split("\n")
    assert head == "CURRENT BROKERS:"
    got = json.loads(body)
    assert got == [{k: v for k, v in b.items()} for b in BROKERS]
    assert body.startswith('[{"rack":"a","port":9092,"host":"h10","id":10}') and body.endswith('{"port":9093,"host":"h18","id":18}]')     # org.json HashMap key order (predicted)
    rc, out, _ = run(cli, "--zk_string", snapshot, "--mode", "PRINT_CURRENT_ASSIGNMENT", "--topics", "test,logs.v2")
    assert rc == 0 and out == "CURRENT ASSIGNMENT:\n" + expected_current(["test", "logs.v2"]) + "\n"


def test_unknown_broker_host_is_an_error_but_unknown_host_to_remove_is_ignored(cli, snapshot):
    rc, out, err = run(cli, "--zk_string", snapshot, "--mode", "PRINT_CURRENT_BROKERS", "--broker_hosts", "h10,nope")
    assert rc != 0 and "Some hostnames could not be found! We found: [10]" in err   # KAG:199-201 (checkPresence=true)
    rc, out, err = run(cli, "--zk_string", snapshot, "--mode", "PRINT_CURRENT_BROKERS", "--broker_hosts_to_remove", "nope")
    assert rc == 0                                                                  # KAG:233 (checkPresence=false)
    rc, out, err = run(cli, "--zk_string", snapshot, "--mode", "PRINT_CURRENT_BROKERS", "--integer_broker_ids", "10,x")
    assert rc != 0 and "Invalid broker ID: x" in err                                # KAG:214-216


# ---- GPU ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_print_reassignment_matches_oracle_json(cli, snapshot):
    all_ids = [b["id"] for b in BROKERS]
    racks = {b["id"]: b["rack"] for b in BROKERS if "rack" in b}

    def check(args, names, brokers, rk, desired=-1):
        rc, out, err = run(cli, "--zk_string", snapshot, "--mode", "PRINT_REASSIGNMENT", *args)
        assert rc == 0, err
        exp = "CURRENT ASSIGNMENT:\n" + expected_current(names) + "\nNEW ASSIGNMENT:\n" + \
              expected_new_assignment(names, brokers, {b: r for b, r in rk.items() if b in brokers}, desired) + "\n"
        assert out == exp

    check([], ORDER, all_ids, racks)                                                   # all topics, all brokers
    check(["--broker_hosts_to_remove", "h12,ghost"], ORDER, [b for b in all_ids if b != 12], racks)   # decommission
    check(["--disable_rack_awareness"], ORDER, all_ids, {})
    check(["--topics", "test,events"], ["test", "events"], all_ids, racks)             # explicit topic order
    check(["--broker_hosts", "h10,h11,h13,h14,h15,h16,h17"], ORDER, [10, 11, 13, 14, 15, 16, 17], racks)
    check(["--integer_broker_ids", "10,11,12,13,14,15,16,17,18", "--desired_replication_factor", "2"], ORDER, all_ids, racks, 2)
    # a run the reference itself cannot finish: same exception text, no NEW ASSIGNMENT
    rc, out, err = run(cli, "--zk_string", snapshot, "--mode", "PRINT_REASSIGNMENT", "--integer_broker_ids", "10,11,12,13,14,15")
    assert rc != 0 and "java.lang.IllegalStateException: Partition 1 could not be fully assigned!" in err and "NEW ASSIGNMENT" not in out


@pytest.mark.gpu
def test_topic_without_partition_records_behaves_like_an_empty_assignment(cli, snapshot):
    """ZkUtils.getPartitionAssignmentForTopics gives an empty map for such a topic (ADVICE r1): KTA:65-66 throws unless
    --desired_replication_factor is given, in which case the topic simply contributes no rows."""
    rc, out, err = run(cli, "--zk_string", snapshot, "--mode", "PRINT_REASSIGNMENT", "--topics", "test,nosuch")
    assert rc != 0 and "java.lang.IllegalStateException: Topic nosuch does not have a positive replication factor!" in err
    assert "NEW ASSIGNMENT" not in out
    rc, out, err = run(cli, "--zk_string", snapshot, "--mode", "PRINT_REASSIGNMENT", "--topics", "test,nosuch",
                       "--desired_replication_factor", "2")
    assert rc == 0, err
    all_ids = [b["id"] for b in BROKERS]
    racks = {b["id"]: b["rack"] for b in BROKERS if "rack" in b}
    assert out.endswith("NEW ASSIGNMENT:\n" + expected_new_assignment(["test"], all_ids, racks, 2) + "\n")


@pytest.mark.gpu
def test_reassignment_errors_abort_without_new_assignment(cli, snapshot):
    rc, out, err = run(cli, "--zk_string", snapshot, "--mode", "PRINT_REASSIGNMENT", "--integer_broker_ids", "10,11")
    assert rc != 0
    assert "NEW ASSIGNMENT" not in out and out.startswith("CURRENT ASSIGNMENT:\n")      # KAG:160 printed, KAG:186 never
    assert "java.lang.IllegalStateException: Topic events has a higher replication factor (3) than available brokers!" in err
    rc, out, err = run(cli, "--zk_string", snapshot, "--mode", "PRINT_REASSIGNMENT", "--topics", "test,missing")
    # a topic without partition records is an EMPTY assignment (ZkUtils), i.e. KTA:65-66 — not the NPE of a null map
    assert rc != 0 and "Topic missing does not have a positive replication factor!" in err and "NEW ASSIGNMENT" not in out


@pytest.mark.gpu
def test_cpp_host_mirror_passes_the_reference_junit_suite(cli):
    """host/test_kafka_topic_assigner.cpp: KafkaTopicAssignerTest.java re-expressed against kassign::KafkaTopicAssigner."""
    r = subprocess.run([kab.build_mod.HOST_TEST], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("OK")


def test_org_json_key_order_prediction():
    """The emitters print object keys in the iteration order of the java.util.HashMap behind org.json 20131018's
    JSONObject (default 16 buckets, JDK >= 8 hash spreading h ^ (h >>> 16); no collisions among our keys) — the
    derivation of SURVEY.md §3.4, recomputed here so the constant order in kassign_host.hpp is not folklore.
    (Still a prediction: no JVM in the image to confirm it.)"""
    from oracle import py_oracle as po

    def bucket(key):
        h = po.java_string_hash(key) & 0xFFFFFFFF
        return (h ^ (h >> 16)) & 15

    assert sorted(["version", "partitions"], key=bucket) == ["partitions", "version"]                 # KAG:169-171,185
    assert sorted(["topic", "partition", "replicas"], key=bucket) == ["partition", "replicas", "topic"]  # KAG:178-182
    assert sorted(["id", "host", "port", "rack"], key=bucket) == ["rack", "port", "host", "id"]        # KAG:117-124
    assert len({bucket(k) for k in ["topic", "partition", "replicas"]}) == 3 and len({bucket(k) for k in ["id", "host", "port", "rack"]}) == 4
