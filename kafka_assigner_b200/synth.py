"""Synthetic cluster generator for the BASELINE.json configs (SURVEY.md §8d).

Deterministic (counter-based splitmix64), numpy-vectorised so config 4 (76.8 M replica slots) is
generated in seconds. The same arrays are fed to the oracle and to the CUDA path.

Reference shapes being synthesised: the inputs of KafkaTopicAssigner.generateAssignment
(KafkaTopicAssigner.java:42-44): per topic `currentAssignment` (partition -> ordered broker list),
the live `brokers` set and the `rackAssignment` map, plus the topic names whose String.hashCode
rotates the processing order (KafkaAssignmentStrategy.java:188-200).
"""
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

_GOLDEN = np.uint64(0x9E3779B97F4A7C15)
_M1 = np.uint64(0xBF58476D1CE4E5B9)
_M2 = np.uint64(0x94D049BB133111EB)


def splitmix64(seed: int, index) -> np.ndarray:
    """Value #index of the splitmix64 stream seeded with `seed` (vectorised over `index`)."""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + (np.asarray(index, dtype=np.uint64) + np.uint64(1)) * _GOLDEN
        z = (z ^ (z >> np.uint64(30))) * _M1
        z = (z ^ (z >> np.uint64(27))) * _M2
        return z ^ (z >> np.uint64(31))


def java_string_hash_ascii(names: List[str]) -> np.ndarray:
    """String.hashCode for ASCII names, vectorised (test/bench convenience; the product uses
    ka_java_string_hash)."""
    out = np.zeros(len(names), dtype=np.uint32)
    for i, n in enumerate(names):
        h = 0
        for ch in n.encode("ascii"):
            h = (h * 31 + ch) & 0xFFFFFFFF
        out[i] = h
    return out.view(np.int32)


@dataclass
class Cluster:
    """A flat, solver-ready problem: T topics, dense P partitions x RF replicas each."""
    name: str
    topic_names: List[str]
    topic_hash: np.ndarray          # int32 [T]
    P: int
    RF: int
    cur: np.ndarray                 # int32 [T, P, RF] broker IDs (leader first)
    broker_id: np.ndarray           # int32 [N] ascending — the LIVE set handed to the solver
    rack_name: List[Optional[str]]  # per live broker
    rack_index: np.ndarray          # int32 [N] dense rack index (string-keyed, KAS:81-94)
    desired_rf: int = -1
    meta: dict = field(default_factory=dict)

    @property
    def T(self):
        return len(self.topic_names)

    @property
    def N(self):
        return len(self.broker_id)

    @property
    def replicas(self):
        return self.T * self.P * self.RF

    def ragged(self):
        """(part_off, part_id, rep_off, cur_flat) for the general ka_solve / oracle entry."""
        T, P, RF = self.T, self.P, self.RF
        part_off = np.arange(T + 1, dtype=np.int64) * P
        part_id = np.tile(np.arange(P, dtype=np.int32), T)
        rep_off = np.arange(T * P + 1, dtype=np.int64) * RF
        return part_off, part_id, rep_off, np.ascontiguousarray(self.cur.reshape(-1))

    def subset(self, t0, t1):
        """Topics [t0, t1) as their own Cluster (same brokers) — topic sharding / bounded CPU samples."""
        return Cluster(self.name + "[%d:%d]" % (t0, t1), self.topic_names[t0:t1], self.topic_hash[t0:t1].copy(),
                       self.P, self.RF, np.ascontiguousarray(self.cur[t0:t1]), self.broker_id, self.rack_name,
                       self.rack_index, self.desired_rf, dict(self.meta))


def rack_indices(broker_id, rack_name):
    """Dense rack index with the reference's string-key semantics (KAS:81-94): key = rack string, or
    str(id) when no rack is defined; equal keys share a rack."""
    keys = {}
    out = np.zeros(len(broker_id), dtype=np.int32)
    for i, (b, r) in enumerate(zip(broker_id, rack_name)):
        k = r if r is not None else str(int(b))
        out[i] = keys.setdefault(k, len(keys))
    return out


def _live_brokers(N, R, remove_frac, rack_aware=True):
    """make_cluster's live set: brokers 1000+i, rack i % R, minus the round(remove_frac*N/R) highest ordinals of every rack."""
    ordinal = np.arange(N)
    per_rack_remove = int(round(remove_frac * N / R))
    rack_of = ordinal % R
    rank_in_rack = ordinal // R
    rack_sizes = np.bincount(rack_of, minlength=R)
    live_mask = rank_in_rack < (rack_sizes[rack_of] - per_rack_remove)
    live_ids = (1000 + ordinal[live_mask]).astype(np.int32)
    return live_ids, ["r%02d" % (i % R) if rack_aware else None for i in ordinal[live_mask]]


def decommission_tables(key, fracs, **over):
    """The live broker tables (broker_id, rack_index) of make_config(key, remove_frac=f) for every f of fracs, without
    generating the cluster: its current assignment does not depend on remove_frac. For one batched candidate solve."""
    kw = dict(CONFIGS[key])
    kw.update(over)
    out = []
    for f in fracs:
        ids, names = _live_brokers(kw["N"], kw["R"], f, kw.get("rack_aware", True))
        out.append((ids, rack_indices(ids, names)))
    return out


def make_cluster(T, P, RF, N, R, seed, kind="mixed", n_old=None, remove_frac=0.0, name=None,
                 rack_aware=True, topic_prefix="topic-", t_offset=0):
    """Expansion / decommission scenario of SURVEY §8d.

    brokers: ids 1000+i, rack of broker i = i % R ("r%02d"); the CURRENT assignment lives on the first
    n_old brokers (default N - R*ceil(N/(5R)): whole rack-rows are new), the solver's live set is all N
    minus, per rack, the round(remove_frac*N/R) highest-ordinal brokers.
    kind: "structured" cur[t,p,r] = old[(s_t + RF*p + r) % n_old]; "random" = RF distinct racks, uniform
    broker inside each, random order; "mixed" = even topics structured, odd topics random.
    t_offset: generate topics [t_offset, t_offset+T) of a longer run (names, hashes and random streams are
    indexed by the GLOBAL topic number, so shards of one job can be generated independently per rank).
    """
    assert R >= RF and N >= R
    if n_old is None:
        n_old = N - R * int(np.ceil(N / (5.0 * R)))
        if n_old < R * 1:
            n_old = N
    n_old = max(R, (n_old // R) * R)
    all_ids = (1000 + np.arange(N)).astype(np.int32)
    live_ids, rack_names = _live_brokers(N, R, remove_frac, rack_aware)

    names = ["%s%06d" % (topic_prefix, t) for t in range(t_offset, t_offset + T)]
    th = java_string_hash_ascii(names)
    assert not np.any(th == np.int32(-2**31)), "synthetic topic name hashes to Integer.MIN_VALUE"

    t_idx = np.arange(t_offset, t_offset + T, dtype=np.uint64)
    s_t = (splitmix64(seed, t_idx) % np.uint64(n_old)).astype(np.int64)  # per-topic offset
    cur = np.empty((T, P, RF), dtype=np.int32)
    p_idx = np.arange(P, dtype=np.int64)
    structured = (s_t[:, None, None] + RF * p_idx[None, :, None] + np.arange(RF)[None, None, :]) % n_old
    if kind == "structured":
        cur[:] = all_ids[structured]
    else:
        # random: RF distinct racks, then a uniform old broker inside each rack
        chunk = max(1, (1 << 22) // max(1, P * RF))
        per_rack_old = n_old // R
        for t0 in range(0, T, chunk):
            t1 = min(T, t0 + chunk)
            tt = np.arange(t_offset + t0, t_offset + t1, dtype=np.uint64)
            base = ((tt[:, None] * np.uint64(P) + np.arange(P, dtype=np.uint64)[None, :]) * np.uint64(16)) + np.uint64(1 << 40)
            racks = np.empty((t1 - t0, P, RF), dtype=np.int64)
            for r in range(RF):
                draw = (splitmix64(seed, base + np.uint64(r)) % np.uint64(R - r)).astype(np.int64)
                # skip the racks already taken (ascending-insert trick)
                taken = np.sort(racks[:, :, :r], axis=2) if r else None
                for j in range(r):
                    draw = draw + (draw >= taken[:, :, j])
                racks[:, :, r] = draw
            within = (splitmix64(seed, base[:, :, None] + np.uint64(8) + np.arange(RF, dtype=np.uint64)[None, None, :])
                      % np.uint64(per_rack_old)).astype(np.int64)
            rnd = all_ids[racks + within * R]
            if kind == "random":
                cur[t0:t1] = rnd
            else:  # mixed
                cur[t0:t1] = all_ids[structured[t0:t1]]
                odd = (np.arange(t_offset + t0, t_offset + t1) % 2) == 1
                cur[t0:t1][odd] = rnd[odd]
    ri = rack_indices(live_ids, rack_names)
    return Cluster(name or "T%d_P%d_RF%d_N%d_R%d_%s" % (T, P, RF, N, R, kind), names, th, P, RF, cur, live_ids,
                   rack_names, ri, -1,
                   dict(T=T, P=P, RF=RF, N=N, R=R, seed=seed, kind=kind, n_old=n_old, remove_frac=remove_frac))


@dataclass
class RaggedCluster:
    """A real-cluster-shaped problem in the ragged layout of ka_solve / ka_solve_json: partition counts and replication
    factors differ from topic to topic."""
    name: str
    topic_names: List[str]
    topic_hash: np.ndarray          # int32 [T]
    part_off: np.ndarray            # int64 [T+1]
    part_id: np.ndarray             # int32 [Q] 0..P_t-1 per topic
    rep_off: np.ndarray             # int64 [Q+1]
    cur: np.ndarray                 # int32 [R] current replica lists, leader first
    broker_id: np.ndarray           # int32 [N] ascending — the LIVE set handed to the solver
    rack_name: List[Optional[str]]  # per live broker (None: no rack defined)
    rack_index: np.ndarray          # int32 [N]
    all_broker_id: np.ndarray       # int32 every broker of the cluster, removed ones included (ascending)
    all_rack_name: List[Optional[str]]
    desired_rf: int = -1
    meta: dict = field(default_factory=dict)

    @property
    def T(self):
        return len(self.topic_names)

    @property
    def Q(self):
        return int(self.part_off[-1])

    @property
    def N(self):
        return len(self.broker_id)

    def topics(self):
        """[(name, {partition: [brokers]})] — the per-topic maps of the reference's generateAssignment loop."""
        out = []
        for t, n in enumerate(self.topic_names):
            a, b = int(self.part_off[t]), int(self.part_off[t + 1])
            out.append((n, {int(self.part_id[g]): self.cur[self.rep_off[g]:self.rep_off[g + 1]].tolist() for g in range(a, b)}))
        return out


def _ragged_live(all_ids, all_racks, seed, remove_frac):
    """make_ragged_cluster's live set: round(remove_frac * N) brokers drawn at random (seeded) leave; (ids, rack names)."""
    N = len(all_ids)
    removed = np.argsort(splitmix64(seed + 5, np.arange(N, dtype=np.uint64)))[:int(round(remove_frac * N))]
    live = np.ones(N, dtype=bool)
    live[removed] = False
    return all_ids[live], [all_racks[i] for i in range(N) if live[i]]


def ragged_decommission_tables(cluster, fracs):
    """The live broker tables (broker_id, rack_index) that make_ragged_cluster(..., remove_frac=f) with cluster's other
    arguments would produce, for every f of fracs, without regenerating the cluster (its lists do not depend on remove_frac).
    For one batched candidate solve."""
    out = []
    for f in fracs:
        ids, racks = _ragged_live(cluster.all_broker_id, cluster.all_rack_name, cluster.meta["seed"], f)
        out.append((ids, rack_indices(ids, racks)))
    return out


def make_ragged_cluster(T, N=800, R=10, seed=0, max_partitions=256, tail=1.1, rf_weights=(0.15, 0.25, 0.6),
                        rack_frac=0.8, new_frac=0.1, remove_frac=0.0, desired_rf=-1, topic_prefix="svc."):
    """A seeded, deterministic real-cluster shape.

    Topic t has P_t = min(max_partitions, floor(u^(-1/tail))) partitions (a Pareto tail: most topics have a handful, a few have
    hundreds) and replication factor 1, 2 or 3 drawn with rf_weights. Brokers are ids 1..N; broker i is in rack "r<i % R>"
    with probability rack_frac and has no rack otherwise. The current lists use the first N - round(new_frac * N) brokers
    (the rest joined empty); remove_frac of the brokers (drawn at random) leave the live set.
    """
    t_idx = np.arange(T, dtype=np.uint64)
    u = (splitmix64(seed, t_idx) >> np.uint64(11)).astype(np.float64) / float(1 << 53)
    P = np.minimum(max_partitions, np.floor((1.0 - u) ** (-1.0 / tail))).astype(np.int64)
    w = np.cumsum(np.asarray(rf_weights, dtype=np.float64) / sum(rf_weights))
    v = (splitmix64(seed + 1, t_idx) >> np.uint64(11)).astype(np.float64) / float(1 << 53)
    rf = (1 + np.searchsorted(w, v, side="right")).clip(1, len(rf_weights)).astype(np.int64)
    part_off = np.zeros(T + 1, dtype=np.int64)
    np.cumsum(P, out=part_off[1:])
    Q = int(part_off[-1])
    topic_of = np.repeat(np.arange(T), P)
    part_id = (np.arange(Q, dtype=np.int64) - part_off[topic_of]).astype(np.int32)
    rf_row = rf[topic_of]
    rep_off = np.zeros(Q + 1, dtype=np.int64)
    np.cumsum(rf_row, out=rep_off[1:])
    # current lists: RF distinct old brokers base, base + step, base + 2 step (mod n_old; 0 < step < n_old / 2)
    all_ids = np.arange(1, N + 1, dtype=np.int32)
    n_old = max(3, N - int(round(new_frac * N)))
    g = np.arange(Q, dtype=np.uint64)
    base = (splitmix64(seed + 2, g) % np.uint64(n_old)).astype(np.int64)
    step = 1 + (splitmix64(seed + 3, g) % np.uint64(max(1, (n_old - 1) // 2))).astype(np.int64)
    slot = np.arange(int(rep_off[-1]), dtype=np.int64) - np.repeat(rep_off[:-1], rf_row)
    cur = all_ids[(np.repeat(base, rf_row) + slot * np.repeat(step, rf_row)) % n_old]
    # racks, removals
    bi = np.arange(N, dtype=np.uint64)
    has_rack = (splitmix64(seed + 4, bi) >> np.uint64(11)).astype(np.float64) / float(1 << 53) < rack_frac
    all_racks = ["r%02d" % (i % R) if has_rack[i] else None for i in range(N)]
    live_ids, live_racks = _ragged_live(all_ids, all_racks, seed, remove_frac)
    names = ["%s%05d" % (topic_prefix, t) for t in range(T)]
    th = java_string_hash_ascii(names)
    assert not np.any(th == np.int32(-2**31)), "synthetic topic name hashes to Integer.MIN_VALUE"
    return RaggedCluster("ragged_T%d_N%d_s%d" % (T, N, seed), names, th, part_off, part_id, rep_off, cur.astype(np.int32),
                         live_ids, live_racks, rack_indices(live_ids, live_racks), all_ids, all_racks, desired_rf,
                         dict(T=T, N=N, R=R, seed=seed, max_partitions=max_partitions, tail=tail, remove_frac=remove_frac))


# BASELINE.json configs (index = position in `configs`); seeds 0x5EED0000 + config#.
CONFIGS = {
    "c1": dict(T=10, P=8, RF=3, N=6, R=3, seed=0x5EED0001, n_old=6),
    "c2": dict(T=1000, P=64, RF=3, N=100, R=10, seed=0x5EED0002),
    "c3": dict(T=10000, P=128, RF=3, N=1000, R=20, seed=0x5EED0003),
    "c4": dict(T=100000, P=256, RF=3, N=5000, R=50, seed=0x5EED0004),
    "c4shard": dict(T=12500, P=256, RF=3, N=5000, R=50, seed=0x5EED0004),  # one GPU's 1/8 of config 4
    "c5": dict(T=1000, P=1000, RF=3, N=10000, R=50, seed=0x5EED0005, n_old=10000),
}


def make_config(key, kind="mixed", **over):
    kw = dict(CONFIGS[key])
    kw.update(over)
    return make_cluster(kind=kind, name=key + "_" + kind, **kw)
