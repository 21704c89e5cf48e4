"""Build libkassign.so (hand-written CUDA for sm_90a) in-tree with nvcc. No JIT cache, no torch."""
import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB = os.path.join(CSRC, "libkassign.so")
SOURCES = ["kassign.cu"]
HEADERS = ["kassign_common.cuh", "kassign_stage.cuh", "kassign_order.cuh", "kassign_json.cuh", "kassign_score.cuh", "kassign_waves.cuh", "kassign_waves_json.cuh", "kassign_usage.cuh", os.path.join("..", "..", "include", "kassign.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-shared", "-Xcompiler", "-fPIC"]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libkassign.so cannot be built (there is no CPU fallback)")


HOST_DIR = os.path.join(_HERE, "host")
CLI = os.path.join(_HERE, "bin", "kafka-assignment-generator")
HOST_TEST = os.path.join(_HERE, "bin", "test_kafka_topic_assigner")
HOST_CANDIDATES_TEST = os.path.join(_HERE, "bin", "test_candidates")
HOST_SCORES_TEST = os.path.join(_HERE, "bin", "test_candidate_scores")
HOST_CLUSTERS_TEST = os.path.join(_HERE, "bin", "test_clusters")
HOST_CLUSTERS_JSON_TEST = os.path.join(_HERE, "bin", "test_clusters_json")
HOST_CLUSTER_SCORES_TEST = os.path.join(_HERE, "bin", "test_cluster_scores")
HOST_WAVES_TEST = os.path.join(_HERE, "bin", "test_waves")
HOST_WAVES_JSON_TEST = os.path.join(_HERE, "bin", "test_waves_json")
HOST_WAVES_SEND_TEST = os.path.join(_HERE, "bin", "test_waves_send")
HOST_WAVE_PARTS_TEST = os.path.join(_HERE, "bin", "test_wave_parts")
HOST_WAVE_ROLLBACK_TEST = os.path.join(_HERE, "bin", "test_wave_rollback")
HOST_BROKER_USAGE_TEST = os.path.join(_HERE, "bin", "test_broker_usage")
HOST_WAVES_FIRST_FIT_TEST = os.path.join(_HERE, "bin", "test_waves_first_fit")
HOST_PART_CAPS_TEST = os.path.join(_HERE, "bin", "test_part_caps")
HOST_SOURCES = ["kafka_assignment_generator.cpp", "kassign_host.hpp", "test_kafka_topic_assigner.cpp", "test_candidates.cpp",
                "test_candidate_scores.cpp", "test_clusters.cpp", "test_clusters_json.cpp", "test_cluster_scores.cpp", "test_waves.cpp", "test_waves_json.cpp",
                "test_waves_send.cpp", "test_wave_parts.cpp", "test_wave_rollback.cpp", "test_broker_usage.cpp", "test_waves_first_fit.cpp",
                "test_part_caps.cpp"]


def build_host(force=False):
    """g++ the C++ host mirror + file-based CLI (reference flag surface) against libkassign.so."""
    deps = [os.path.join(HOST_DIR, f) for f in HOST_SOURCES] + [LIB, os.path.join(_HERE, "..", "include", "kassign.h")]
    if not force and all(os.path.exists(x) for x in (CLI, HOST_TEST, HOST_CANDIDATES_TEST, HOST_SCORES_TEST, HOST_CLUSTERS_TEST,
                                                                   HOST_CLUSTERS_JSON_TEST, HOST_CLUSTER_SCORES_TEST, HOST_WAVES_TEST, HOST_WAVES_JSON_TEST, HOST_WAVES_SEND_TEST, HOST_WAVE_PARTS_TEST, HOST_WAVE_ROLLBACK_TEST, HOST_BROKER_USAGE_TEST, HOST_WAVES_FIRST_FIT_TEST, HOST_PART_CAPS_TEST)) and all(os.path.getmtime(d) <= os.path.getmtime(CLI) for d in deps if os.path.exists(d)):
        return CLI
    os.makedirs(os.path.dirname(CLI), exist_ok=True)
    cmd = ["g++", "-O2", "-std=c++17", "-Wall", os.path.join(HOST_DIR, "kafka_assignment_generator.cpp"), "-L" + CSRC, "-lkassign",
           "-Wl,-rpath,$ORIGIN/../csrc", "-o", CLI]
    subprocess.check_call(cmd)
    for src, exe in (("test_kafka_topic_assigner.cpp", HOST_TEST), ("test_candidates.cpp", HOST_CANDIDATES_TEST),
                     ("test_candidate_scores.cpp", HOST_SCORES_TEST), ("test_clusters.cpp", HOST_CLUSTERS_TEST),
                     ("test_clusters_json.cpp", HOST_CLUSTERS_JSON_TEST), ("test_cluster_scores.cpp", HOST_CLUSTER_SCORES_TEST),
                     ("test_waves.cpp", HOST_WAVES_TEST), ("test_waves_json.cpp", HOST_WAVES_JSON_TEST),
                     ("test_waves_send.cpp", HOST_WAVES_SEND_TEST), ("test_wave_parts.cpp", HOST_WAVE_PARTS_TEST),
                     ("test_wave_rollback.cpp", HOST_WAVE_ROLLBACK_TEST), ("test_broker_usage.cpp", HOST_BROKER_USAGE_TEST),
                     ("test_waves_first_fit.cpp", HOST_WAVES_FIRST_FIT_TEST), ("test_part_caps.cpp", HOST_PART_CAPS_TEST)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", os.path.join(HOST_DIR, src), "-L" + CSRC, "-lkassign",
                               "-Wl,-rpath,$ORIGIN/../csrc", "-o", exe])
    return CLI


def needs_build():
    if not os.path.exists(LIB):
        return True
    lib_m = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]  # flags live here
    return any(os.path.getmtime(d) > lib_m for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    """Compile every CUDA source into csrc/libkassign.so. Cross-compiles without a GPU."""
    if not force and not needs_build():
        return LIB
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + SOURCES
    subprocess.check_call(cmd, cwd=CSRC)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
