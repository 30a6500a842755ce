"""Deterministic synthetic pending queues + node tables (SURVEY.md §8d).

The same generated tables feed the CUDA path and (in tests/bench) the oracle.
Seeds are `0xC0FFEE00 + config_id`; `now` = 1_700_000_000. Request views are
derived the way the reference derives them at submit time
(CtldPublicDefs.cpp:1655-1682: cpus_per_task / mem_per_cpu -> req_task_res_view,
gres_per_node -> req_node_res_view; JobScheduler.cpp:6075-6110:
ntasks_per_node bounds and req_total_res_view = node*node_num + task*ntasks).
Node totals follow CranedMetaContainer.cpp:318-346 (cores {0..n-1},
cpu = n, mem_sw = mem, configured gres slots).
"""
from __future__ import annotations

import numpy as np

from .abi import (CORE_WORDS, GRES_ENTRIES, RES_IN_NODE, RES_VIEW, Cluster, Config,
                  Pending, Running)

NOW = 1_700_000_000
GiB = 1 << 30
DAY = 24 * 3600
SEED_BASE = 0xC0FFEE00


def _rng(config_id: int, salt: int = 0) -> np.random.Generator:
    return np.random.Generator(np.random.PCG64(SEED_BASE + config_id + (salt << 32)))


def node_row(cores: int, mem: int, gres: dict[int, int] | None = None) -> np.ndarray:
    """res_total of one node: cores {0..n-1}; gres = {entry: n_slots}."""
    r = np.zeros((), RES_IN_NODE)
    r["cpu_raw"] = cores * 256
    r["mem"] = mem
    r["mem_sw"] = mem
    for w in range(CORE_WORDS):
        k = min(max(cores - 64 * w, 0), 64)
        r["core"][w] = (1 << k) - 1 if k < 64 else 0xFFFFFFFFFFFFFFFF
    for e, n in (gres or {}).items():
        r["gres"][e] = (1 << n) - 1
    return r


def make_cluster(groups, gres_entry_name=()) -> Cluster:
    """groups: list of (count, node_row) -> one disjoint partition per group."""
    rows, off, nodes = [], [0], []
    base = 0
    for count, row in groups:
        rows.append(np.repeat(row[None], count))
        nodes.append(np.arange(base, base + count, dtype=np.uint32))
        base += count
        off.append(base)
    res_total = np.concatenate(rows)
    m = len(res_total)
    return Cluster(res_total, np.ones(m, np.uint8), np.zeros(m, np.uint8),
                   np.array(off, np.uint32), np.concatenate(nodes),
                   len(gres_entry_name), tuple(gres_entry_name))


def _views(n, cpus_raw, mem_per_task, node_num, ntasks, gres_total=None, gres_spec=None,
           mem_per_node=None):
    req_node = np.zeros(n, RES_VIEW)
    req_task = np.zeros(n, RES_VIEW)
    req_task["cpu_raw"] = cpus_raw
    req_task["mem"] = mem_per_task
    req_task["mem_sw"] = mem_per_task
    if mem_per_node is not None:
        req_node["mem"] = mem_per_node
        req_node["mem_sw"] = mem_per_node
    if gres_total is not None:
        req_node["gres_total"] = gres_total
    if gres_spec is not None:
        req_node["gres_spec"] = gres_spec
    req_total = np.zeros(n, RES_VIEW)
    nn = node_num.astype(np.int64)
    nt = ntasks.astype(np.int64)
    for f in ("cpu_raw", "mem", "mem_sw"):
        req_total[f] = (req_node[f].astype(np.int64) * nn + req_task[f].astype(np.int64) * nt).astype(req_total[f].dtype)
    for f in ("gres_total", "gres_spec"):
        req_total[f] = (req_node[f].astype(np.int64) * nn[:, None]
                        + req_task[f].astype(np.int64) * nt[:, None]).astype(np.uint16)
    return req_node, req_task, req_total


def _log_uniform(rng, lo, hi, n):
    return np.exp(rng.uniform(np.log(lo), np.log(hi), n)).astype(np.int64)


def _pending(n, partition, time_limit, submit, node_num, ntasks, views, part_prio, qos_prio,
             account=None, qos=None, user=None, exclusive=None, ntpn=None, mandated=None,
             incl=None, excl=None):
    z32 = np.zeros(n, np.uint32)
    ntpn_min, ntpn_max = ntpn if ntpn is not None else (np.ones(n, np.uint32), np.ones(n, np.uint32))
    req_node, req_task, req_total = views
    kw = {}
    if incl is not None:
        kw.update(incl_off=incl[0], incl_nodes=incl[1])
    if excl is not None:
        kw.update(excl_off=excl[0], excl_nodes=excl[1])
    return Pending(
        partition, time_limit, submit, node_num, ntasks, ntpn_min, ntpn_max,
        exclusive if exclusive is not None else np.zeros(n, np.uint8),
        part_prio, qos_prio,
        account if account is not None else z32, qos if qos is not None else z32,
        user if user is not None else z32,
        mandated if mandated is not None else np.zeros(n, np.float64),
        req_node, req_task, req_total, **kw)


# ---------------------------------------------------------------------------
# Config 1: 1k x 128, cpu+mem, single partition, FIFO
# ---------------------------------------------------------------------------
def config1(n_jobs=1000, n_nodes=128):
    rng = _rng(1)
    cluster = make_cluster([(n_nodes, node_row(64, 256 * GiB))])
    cpus = rng.choice([1, 2, 4, 8], n_jobs)
    node_num = np.ones(n_jobs, np.uint32)
    views = _views(n_jobs, cpus * 256, cpus.astype(np.uint64) * 2 * GiB, node_num, node_num)
    pend = _pending(n_jobs, np.zeros(n_jobs, np.uint32), rng.integers(60, 3601, n_jobs),
                    np.full(n_jobs, NOW - 100, np.int64), node_num, node_num, views,
                    np.full(n_jobs, 1000, np.uint32), np.full(n_jobs, 1000, np.uint32))
    cfg = Config(priority_type=0, scheduled_batch_size=100_000)
    return cfg, cluster, Running.empty(), pend, NOW


# ---------------------------------------------------------------------------
# Config 2: 100k x 10k, cpu+mem+gres(GPU), 4 partitions, multifactor+backfill
# ---------------------------------------------------------------------------
CONFIG2_WEIGHTS = dict(weight_age=500, weight_fair_share=10000, weight_job_size=0,
                       weight_partition=1000, weight_qos=1_000_000, favor_small=True,
                       max_age_s=7 * DAY)  # etc/config.yaml:96-106


def config2(n_jobs=100_000, n_nodes=10_000, seed_id=2, limit=None):
    rng = _rng(seed_id)
    frac = np.array([0.4, 0.3, 0.2, 0.1])
    counts = np.maximum((frac * n_nodes).astype(int), 1)
    groups = [
        (counts[0], node_row(64, 256 * GiB)),
        (counts[1], node_row(128, 512 * GiB)),
        (counts[2], node_row(64, 512 * GiB, {0: 8})),    # gpu:a100 x8
        (counts[3], node_row(96, 1024 * GiB, {1: 8})),   # gpu:h100 x8
    ]
    cluster = make_cluster(groups, gres_entry_name=(0, 0))
    part = rng.choice(4, n_jobs, p=counts / counts.sum()).astype(np.uint32)
    node_num = rng.choice([1, 2, 4, 8], n_jobs, p=[0.85, 0.08, 0.05, 0.02]).astype(np.uint32)
    cpus = rng.choice([1, 2, 4, 8, 16, 32], n_jobs)
    mem_per_cpu = rng.integers(2, 5, n_jobs).astype(np.uint64) * GiB
    gpus = rng.choice([1, 2, 4, 8], n_jobs)
    typed = rng.random(n_jobs) < 0.5
    is_gpu = part >= 2
    gres_total = np.zeros((n_jobs, 8), np.uint16)
    gres_spec = np.zeros((n_jobs, GRES_ENTRIES), np.uint16)
    gres_total[is_gpu, 0] = gpus[is_gpu]
    ent = (part - 2).clip(0, 1)
    sel = is_gpu & typed
    gres_spec[np.flatnonzero(sel), ent[sel]] = gpus[sel]
    views = _views(n_jobs, cpus * 256, cpus.astype(np.uint64) * mem_per_cpu, node_num, node_num,
                   gres_total, gres_spec)
    part_prio = np.array([1000, 2000, 3000, 4000], np.uint32)[part]
    pend = _pending(n_jobs, part, _log_uniform(rng, 60, 48 * 3600, n_jobs),
                    NOW - rng.integers(0, 7 * DAY + 1, n_jobs), node_num, node_num, views,
                    part_prio, rng.choice([1000, 2000, 5000], n_jobs).astype(np.uint32),
                    account=rng.integers(0, 64, n_jobs).astype(np.uint32),
                    qos=rng.integers(0, 3, n_jobs).astype(np.uint32),
                    user=rng.integers(0, 512, n_jobs).astype(np.uint32))
    cfg = Config(priority_type=1, scheduled_batch_size=limit or n_jobs, **CONFIG2_WEIGHTS)
    return cfg, cluster, Running.empty(), pend, NOW


# ---------------------------------------------------------------------------
# Config 3: 1M x 50k, 16 partitions (QoS/account ids carried; limit lifted)
# ---------------------------------------------------------------------------
def config3(n_jobs=1_000_000, n_nodes=50_000, n_parts=16, seed_id=3):
    rng = _rng(seed_id)
    per = n_nodes // n_parts
    kinds = [node_row(64, 256 * GiB), node_row(128, 512 * GiB),
             node_row(64, 512 * GiB, {0: 8}), node_row(96, 1024 * GiB, {1: 8})]
    groups = [(per, kinds[p % 4]) for p in range(n_parts)]
    cluster = make_cluster(groups, gres_entry_name=(0, 0))
    part = rng.integers(0, n_parts, n_jobs).astype(np.uint32)
    node_num = rng.choice([1, 2, 4, 8], n_jobs, p=[0.85, 0.08, 0.05, 0.02]).astype(np.uint32)
    cpus = rng.choice([1, 2, 4, 8, 16, 32], n_jobs)
    mem_per_cpu = rng.integers(2, 5, n_jobs).astype(np.uint64) * GiB
    gpus = rng.choice([1, 2, 4, 8], n_jobs)
    kind = part % 4
    is_gpu = kind >= 2
    typed = rng.random(n_jobs) < 0.5
    gres_total = np.zeros((n_jobs, 8), np.uint16)
    gres_spec = np.zeros((n_jobs, GRES_ENTRIES), np.uint16)
    gres_total[is_gpu, 0] = gpus[is_gpu]
    sel = is_gpu & typed
    gres_spec[np.flatnonzero(sel), (kind[sel] - 2)] = gpus[sel]
    views = _views(n_jobs, cpus * 256, cpus.astype(np.uint64) * mem_per_cpu, node_num, node_num,
                   gres_total, gres_spec)
    pend = _pending(n_jobs, part, _log_uniform(rng, 60, 48 * 3600, n_jobs),
                    NOW - rng.integers(0, 7 * DAY + 1, n_jobs), node_num, node_num, views,
                    (1000 * (1 + part % 4)).astype(np.uint32),
                    rng.choice([1000, 2000, 5000], n_jobs).astype(np.uint32),
                    account=rng.integers(0, 64, n_jobs).astype(np.uint32),
                    qos=rng.integers(0, 8, n_jobs).astype(np.uint32),
                    user=rng.integers(0, 512, n_jobs).astype(np.uint32))
    cfg = Config(priority_type=1, scheduled_batch_size=n_jobs, **CONFIG2_WEIGHTS)
    return cfg, cluster, Running.empty(), pend, NOW


# ---------------------------------------------------------------------------
# Config 4: 500k x 20k heterogeneous gres (GPU/NPU), two gres names per job
# ---------------------------------------------------------------------------
def config4(n_jobs=500_000, n_nodes=20_000, seed_id=4):
    rng = _rng(seed_id)
    # dictionary: gpu:{a100,h100,l40} = entries 0..2 (name 0); npu:{910b,310p} = 3..4 (name 1)
    names = (0, 0, 0, 1, 1)
    per = n_nodes // 5
    groups = [
        (per, node_row(64, 512 * GiB, {0: 8})),
        (per, node_row(96, 1024 * GiB, {1: 8, 3: 8})),
        (per, node_row(64, 256 * GiB, {2: 4, 0: 4})),
        (per, node_row(128, 1024 * GiB, {3: 16})),
        (n_nodes - 4 * per, node_row(64, 512 * GiB, {4: 8, 2: 8})),
    ]
    cluster = make_cluster(groups, gres_entry_name=names)
    part = rng.integers(0, 5, n_jobs).astype(np.uint32)
    node_num = rng.choice([1, 2, 4], n_jobs, p=[0.9, 0.07, 0.03]).astype(np.uint32)
    cpus = rng.choice([1, 2, 4, 8, 16], n_jobs)
    gres_total = np.zeros((n_jobs, 8), np.uint16)
    gres_spec = np.zeros((n_jobs, GRES_ENTRIES), np.uint16)
    part_entries = {0: [0], 1: [1, 3], 2: [2, 0], 3: [3], 4: [4, 2]}
    for p, ents in part_entries.items():
        idx = np.flatnonzero(part == p)
        for e in ents:
            use = rng.random(len(idx)) < (0.8 if e == ents[0] else 0.4)
            cnt = rng.choice([1, 2, 4], len(idx)).astype(np.uint16)
            typed = rng.random(len(idx)) < 0.5
            gres_total[idx[use], names[e]] += cnt[use]
            gres_spec[idx[use & typed], e] += cnt[use & typed]
    views = _views(n_jobs, cpus * 256, cpus.astype(np.uint64) * 2 * GiB, node_num, node_num,
                   gres_total, gres_spec)
    pend = _pending(n_jobs, part, _log_uniform(rng, 60, 24 * 3600, n_jobs),
                    NOW - rng.integers(0, 7 * DAY + 1, n_jobs), node_num, node_num, views,
                    np.full(n_jobs, 1000, np.uint32),
                    rng.choice([1000, 2000, 5000], n_jobs).astype(np.uint32))
    cfg = Config(priority_type=1, scheduled_batch_size=n_jobs, cost_policy=1, **CONFIG2_WEIGHTS)  # best-fit selection
    return cfg, cluster, Running.empty(), pend, NOW


# ---------------------------------------------------------------------------
# Config 5: backfill stress, 200k x 5k, one partition, wide walltimes
# ---------------------------------------------------------------------------
def config5(n_jobs=200_000, n_nodes=5_000, seed_id=5):
    rng = _rng(seed_id)
    cluster = make_cluster([(n_nodes, node_row(64, 256 * GiB))])
    node_num = np.minimum(rng.zipf(2.0, n_jobs), 64).astype(np.uint32)
    cpus = rng.choice([1, 2, 4, 8, 16, 32, 64], n_jobs)
    views = _views(n_jobs, cpus * 256, cpus.astype(np.uint64) * 2 * GiB, node_num, node_num)
    pend = _pending(n_jobs, np.zeros(n_jobs, np.uint32), _log_uniform(rng, 11, 7 * DAY, n_jobs),
                    NOW - rng.integers(0, 7 * DAY + 1, n_jobs), node_num, node_num, views,
                    np.full(n_jobs, 1000, np.uint32),
                    rng.choice([1000, 2000, 5000], n_jobs).astype(np.uint32))
    cfg = Config(priority_type=1, scheduled_batch_size=n_jobs, **CONFIG2_WEIGHTS)
    return cfg, cluster, Running.empty(), pend, NOW


# ---------------------------------------------------------------------------
# Feature-rich small random case for parity tests: running jobs, fractional
# cpus, typed/untyped gres over two names, include/exclude lists, exclusive
# jobs, dead/drained nodes, unknown partitions, mandated priorities.
# ---------------------------------------------------------------------------
def random_case(seed, n_jobs=300, n_nodes=48, n_parts=3, n_running=40, fifo=False,
                frac_cpu=True, lists=True, exclusive=True, limit=None,
                max_jobs_per_node=1000, short=False, one_type_per_name=False, ntpn_range=False, cost_policy=0):
    """one_type_per_name: no node carries two types of the same gres name, so the
    reference's unordered_map walk over a node's types (PublicHeader.cpp:564,583)
    has a single possible order — the cases oracle/_ref can pin (tests/test_ref_pin.py)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    names = (0, 0, 1)  # gpu:a, gpu:b, npu:x
    kinds = [node_row(16, 64 * GiB), node_row(32, 128 * GiB, {0: 4, 1: 4}),
             node_row(24, 96 * GiB, {0: 2, 2: 8}), node_row(8, 32 * GiB, {1: 8})]
    if one_type_per_name:
        kinds[1] = node_row(32, 128 * GiB, {0: 4, 2: 4})
    sizes = rng.multinomial(n_nodes - n_parts, np.ones(n_parts) / n_parts) + 1
    rows, off, base = [], [0], 0
    for p in range(n_parts):
        k = rng.integers(0, len(kinds), sizes[p])
        rows.append(np.stack([kinds[i] for i in k]))
        base += sizes[p]
        off.append(base)
    res_total = np.concatenate(rows)
    alive = (rng.random(n_nodes) > 0.05).astype(np.uint8)
    drain = (rng.random(n_nodes) < 0.05).astype(np.uint8)
    cluster = Cluster(res_total, alive, drain, np.array(off, np.uint32),
                      np.arange(n_nodes, dtype=np.uint32), len(names), names)
    node_part = np.repeat(np.arange(n_parts), sizes)

    def gres_req(n, parts):
        tot = np.zeros((n, 8), np.uint16)
        spec = np.zeros((n, GRES_ENTRIES), np.uint16)
        for i in range(n):
            if rng.random() < 0.5:
                continue
            for g, ents in ((0, (0, 1)), (1, (2,))):
                if rng.random() < 0.5:
                    continue
                t = 0
                for e in ents:
                    if rng.random() < 0.4:
                        c = int(rng.integers(1, 4))
                        spec[i, e] = c
                        t += c
                tot[i, g] = t + (int(rng.integers(0, 3)) if rng.random() < 0.6 else 0)
                if tot[i, g] == 0:
                    tot[i, g] = 1
        return tot, spec

    # running jobs: carve allocations out of node totals with a host-side
    # first-fit so that they are consistent (alloc <= what is left).
    left = res_total.copy()
    r_start, r_end, r_nn, r_pp, r_qp, r_acc, r_cpu, r_mem = [], [], [], [], [], [], [], []
    r_off, r_node, r_res = [0], [], []
    for _ in range(n_running):
        nn = int(rng.choice([1, 1, 1, 2]))
        nodes = rng.choice(n_nodes, nn, replace=False)
        ok_nodes, rowsj = [], []
        for nd in nodes:
            cores = int(rng.integers(1, 5))
            row = np.zeros((), RES_IN_NODE)
            avail_bits = [b for b in range(64) if int(left[nd]["core"][0]) >> b & 1]
            mem = int(rng.integers(1, 9)) * GiB
            if len(avail_bits) < cores or int(left[nd]["mem"]) < mem:
                continue
            if frac_cpu and rng.random() < 0.2:
                row["cpu_raw"] = cores * 256 - 128  # fractional: no cores bound
            else:
                row["cpu_raw"] = cores * 256
                m = 0
                for b in avail_bits[:cores]:
                    m |= 1 << b
                row["core"][0] = m
            row["mem"] = mem
            row["mem_sw"] = mem
            for e in range(len(names)):
                have = int(left[nd]["gres"][e])
                if have and rng.random() < 0.4:
                    low = have & -have
                    row["gres"][e] = low
            if int(left[nd]["cpu_raw"]) < int(row["cpu_raw"]):
                continue
            left[nd]["cpu_raw"] -= row["cpu_raw"]
            left[nd]["mem"] -= row["mem"]
            left[nd]["mem_sw"] -= row["mem_sw"]
            left[nd]["core"][0] &= ~row["core"][0]
            left[nd]["gres"] &= ~row["gres"]
            ok_nodes.append(nd)
            rowsj.append(row)
        if not ok_nodes:
            continue
        order = np.argsort(ok_nodes)
        for o in order:
            r_node.append(ok_nodes[o])
            r_res.append(rowsj[o])
        r_off.append(len(r_node))
        st = NOW - int(rng.integers(1, 5000))
        r_start.append(st)
        r_end.append(NOW + int(rng.integers(-10, 20000)))
        r_nn.append(len(ok_nodes))
        r_pp.append(int(rng.choice([1000, 2000])))
        r_qp.append(int(rng.choice([1000, 5000])))
        r_acc.append(int(rng.integers(0, 6)))
        r_cpu.append(sum(int(r["cpu_raw"]) for r in rowsj))
        r_mem.append(sum(int(r["mem"]) for r in rowsj))
    running = Running(r_start, r_end, r_nn, r_pp, r_qp, r_acc, r_cpu, r_mem, r_off,
                      np.array(r_node, np.uint32),
                      np.array(r_res, RES_IN_NODE) if r_res else np.zeros(0, RES_IN_NODE))

    part = rng.integers(0, n_parts, n_jobs).astype(np.uint32)
    part[rng.random(n_jobs) < 0.02] = n_parts + 3  # "Partition Not Found"
    node_num = rng.choice([1, 1, 1, 2, 3, 5], n_jobs).astype(np.uint32)
    cpus_raw = rng.choice([1, 1, 2, 2, 4, 8, 16], n_jobs) * 256
    if frac_cpu:
        fr = rng.random(n_jobs) < 0.15
        cpus_raw[fr] = rng.choice([64, 128, 384, 640], int(fr.sum()))
    tpn = np.ones(n_jobs, np.uint32)
    multi = rng.random(n_jobs) < 0.2
    tpn[multi] = rng.integers(2, 4, int(multi.sum()))
    ntasks = node_num * tpn
    tpn_max = tpn.copy()
    if ntpn_range:  # general task distribution: ntasks anywhere in [node_num*min, node_num*max]
        wide = rng.random(n_jobs) < 0.5
        tpn_max[wide] = tpn[wide] + rng.integers(1, 4, int(wide.sum()))
        ntasks = (node_num * tpn + rng.integers(0, 1 << 30, n_jobs) % (node_num * (tpn_max - tpn) + 1)).astype(np.uint32)
    gt, gs = gres_req(n_jobs, part)
    mem_task = rng.integers(1, 9, n_jobs).astype(np.uint64) * GiB // 2
    mem_node = np.where(rng.random(n_jobs) < 0.2, rng.integers(0, 4, n_jobs), 0).astype(np.uint64) * GiB
    views = _views(n_jobs, cpus_raw, mem_task, node_num, ntasks, gt, gs, mem_node)
    excl_flag = ((rng.random(n_jobs) < 0.05) & exclusive).astype(np.uint8)
    incl = excl = None
    if lists:
        io, inodes, eo, enodes = [0], [], [0], []
        for i in range(n_jobs):
            p = part[i]
            cand = np.flatnonzero(node_part == p) if p < n_parts else np.zeros(0, int)
            if len(cand) and rng.random() < 0.08:
                k = int(rng.integers(int(node_num[i]), len(cand) + 1)) if len(cand) >= node_num[i] else len(cand)
                inodes += sorted(rng.choice(cand, max(k, 1), replace=False).tolist())
            io.append(len(inodes))
            if len(cand) and rng.random() < 0.08:
                k = int(rng.integers(1, max(2, len(cand) // 2)))
                enodes += sorted(rng.choice(cand, k, replace=False).tolist())
            eo.append(len(enodes))
        incl = (np.array(io, np.uint32), np.array(inodes, np.uint32))
        excl = (np.array(eo, np.uint32), np.array(enodes, np.uint32))
    mand = np.where(rng.random(n_jobs) < 0.03, rng.uniform(1, 2e6, n_jobs), 0.0)
    tl = _log_uniform(rng, 11, 3600 if short else 9 * DAY, n_jobs)
    pend = _pending(n_jobs, part, tl, NOW - rng.integers(0, 9 * DAY, n_jobs), node_num, ntasks,
                    views, rng.choice([1000, 2000, 3000], n_jobs).astype(np.uint32),
                    rng.choice([1000, 2000, 5000], n_jobs).astype(np.uint32),
                    account=rng.integers(0, 6, n_jobs).astype(np.uint32),
                    qos=rng.integers(0, 3, n_jobs).astype(np.uint32),
                    user=rng.integers(0, 20, n_jobs).astype(np.uint32),
                    exclusive=excl_flag, ntpn=(tpn, tpn_max), mandated=mand,
                    incl=incl, excl=excl)
    cfg = Config(priority_type=0 if fifo else 1, scheduled_batch_size=limit or n_jobs,
                 max_jobs_per_node=max_jobs_per_node, cost_policy=cost_policy,
                 weight_age=500, weight_fair_share=10000, weight_job_size=300,
                 weight_partition=1000, weight_qos=1_000_000, favor_small=bool(seed & 1))
    return cfg, cluster, running, pend, NOW


# ---------------------------------------------------------------------------
# Cases at the kernels' size limits: many node shapes per partition, cores up to
# 256 (not always a prefix), all eight gres entries with up to 16 slots, jobs
# wider than a batch (32), than one re-key (64) and up to the general task
# distribution's heap (127 nodes), running jobs holding high cores and slots.
# ---------------------------------------------------------------------------
EDGE_CORES = (8, 32, 64, 65, 96, 128, 129, 192, 255, 256)
EDGE_WIDE = (31, 32, 33, 63, 64, 65, 100, 127)
EDGE_SLOTS = (1, 2, 4, 8, 12, 16)


def _bits_mask(bits, words):
    m = [0] * words
    for b in bits:
        m[b // 64] |= 1 << (b % 64)
    return m


def _edge_shape(rng, k, n_entries):
    """One res_total row; k (the shape's index) makes rows of different shapes distinct."""
    cores = int(rng.choice(EDGE_CORES))
    u = rng.random()
    if u < 0.25 and cores < 256:  # a run of cores that does not start at 0
        lo = int(rng.integers(1, 256 - cores + 1))
        bits = range(lo, lo + cores)
    elif u < 0.4:  # scattered over all four words
        bits = rng.choice(256, cores, replace=False).tolist()
    else:
        bits = range(cores)
    r = np.zeros((), RES_IN_NODE)
    r["cpu_raw"] = cores * 256
    r["mem"] = r["mem_sw"] = (64 + 8 * k) * GiB
    r["core"] = np.array(_bits_mask(bits, CORE_WORDS), np.uint64)
    for e in range(n_entries):
        if rng.random() < 0.55:
            n = int(rng.choice(EDGE_SLOTS))
            slots = range(n) if rng.random() < 0.7 else rng.choice(16, n, replace=False).tolist()
            r["gres"][e] = _bits_mask(slots, 1)[0]
    return r


def _first_bits(mask_words, width, k):
    """The k lowest set bits of a mask given as `width`-bit words (first fit)."""
    out = []
    for w, v in enumerate(mask_words):
        v = int(v)
        while v and len(out) < k:
            low = v & -v
            out.append(w * width + low.bit_length() - 1)
            v ^= low
    return out


def edge_case(seed, n_jobs=400, parts=((140, 20),), one_type_per_name=False, n_running=40,
              wide=EDGE_WIDE, p_wide=0.1, p_general=0.4, p_full=0.01, p_down=0.04, fifo=False, cost_policy=0,
              short=False, limit=None):
    """A case at the kernels' size limits, in the (cfg, cluster, running, pending, now) form of the others.

    parts: (nodes, distinct res_total rows) per partition, disjoint; every shape has at least one usable
    node, so a partition's number of usable classes is exactly its shape count. Gres: eight entries, one
    type per name (one_type_per_name, the layout the reference pin needs) or several types per name.
    Jobs: mostly 1-3 nodes with `p_wide` of them as wide as `wide`, `p_full` as wide as their whole
    partition; `p_general` of the jobs up to 127 nodes get a ntasks_per_node range and uneven ntasks.
    `p_down` of the nodes are dead and as many drained.
    Running jobs are carved first-fit from the node totals (high cores, entries 4-7), some ending inside
    the backfill window. Multifactor priorities are all distinct (mandated): the reference's sort is
    unstable."""
    rng = np.random.Generator(np.random.PCG64(seed))
    names = tuple(range(GRES_ENTRIES)) if one_type_per_name else (0, 0, 0, 1, 1, 1, 2, 2)
    rows, alive, drain, off, sizes, k0 = [], [], [], [0], [], 0
    for n, n_shapes in parts:
        assert 1 <= n_shapes <= n
        shapes = [_edge_shape(rng, k0 + k, GRES_ENTRIES) for k in range(n_shapes)]
        k0 += n_shapes
        pick = np.concatenate([np.arange(n_shapes), rng.integers(0, n_shapes, n - n_shapes)])
        rng.shuffle(pick)
        a = (rng.random(n) >= p_down).astype(np.uint8)
        d = (rng.random(n) < p_down).astype(np.uint8)
        for k in range(n_shapes):  # one usable node of every shape
            first = int(np.flatnonzero(pick == k)[0])
            a[first], d[first] = 1, 0
        rows += [shapes[k] for k in pick]
        alive.append(a)
        drain.append(d)
        sizes.append(n)
        off.append(off[-1] + n)
    res_total = np.array(rows, RES_IN_NODE)
    n_nodes, n_parts = len(res_total), len(parts)
    alive, drain = np.concatenate(alive), np.concatenate(drain)
    cluster = Cluster(res_total, alive, drain, np.array(off, np.uint32), np.arange(n_nodes, dtype=np.uint32),
                      len(names), names)
    usable = [int(((alive == 1) & (drain == 0))[off[p]:off[p + 1]].sum()) for p in range(n_parts)]

    # running jobs: first fit out of what is left on the node, cores of every word, slots of every entry
    left = res_total.copy()
    r_start, r_end, r_nn, r_cpu, r_mem, r_off, r_node, r_res = [], [], [], [], [], [0], [], []
    for _ in range(n_running):
        nn = int(rng.choice([1, 1, 1, 2, 3, 6]))
        ok_nodes, rowsj = [], []
        for nd in sorted(rng.choice(n_nodes, nn, replace=False).tolist()):
            free = _first_bits(left[nd]["core"], 64, 256)
            cores = int(rng.integers(1, 9)) if rng.random() < 0.5 else int(rng.integers(40, 200))
            cores = min(cores, len(free) - 1)
            mem = int(rng.integers(1, 17)) * GiB
            if cores < 1 or int(left[nd]["mem"]) < mem:
                continue
            row = np.zeros((), RES_IN_NODE)
            row["cpu_raw"] = cores * 256
            row["core"] = np.array(_bits_mask(free[:cores], CORE_WORDS), np.uint64)
            row["mem"] = row["mem_sw"] = mem
            for e in range(GRES_ENTRIES):
                have = _first_bits([left[nd]["gres"][e]], 16, 16)
                if have and rng.random() < 0.5:
                    row["gres"][e] = _bits_mask(have[:int(rng.integers(1, len(have) + 1))], 1)[0]
            left[nd]["cpu_raw"] -= row["cpu_raw"]
            left[nd]["mem"] -= row["mem"]
            left[nd]["mem_sw"] -= row["mem_sw"]
            left[nd]["core"] &= ~row["core"]
            left[nd]["gres"] &= ~row["gres"]
            ok_nodes.append(nd)
            rowsj.append(row)
        if not ok_nodes:
            continue
        r_node += ok_nodes
        r_res += rowsj
        r_off.append(len(r_node))
        r_start.append(NOW - int(rng.integers(1, 5000)))
        r_end.append(NOW + int(rng.integers(-10, 3 * DAY if rng.random() < 0.7 else 9 * DAY)))
        r_nn.append(len(ok_nodes))
        r_cpu.append(sum(int(r["cpu_raw"]) for r in rowsj))
        r_mem.append(sum(int(r["mem"]) for r in rowsj))
    k = len(r_start)
    running = Running(r_start, r_end, r_nn, rng.choice([1000, 2000], k), rng.choice([1000, 5000], k),
                      rng.integers(0, 6, k), r_cpu, r_mem, r_off, np.array(r_node, np.uint32),
                      np.array(r_res, RES_IN_NODE) if r_res else np.zeros(0, RES_IN_NODE))

    part = rng.integers(0, n_parts, n_jobs).astype(np.uint32)
    cap = np.array(usable)[part]
    node_num = rng.choice([1, 1, 1, 1, 2, 2, 3], n_jobs)
    w = rng.random(n_jobs) < p_wide
    node_num[w] = np.minimum(rng.choice(wide, int(w.sum())), cap[w])
    full = rng.random(n_jobs) < p_full
    node_num[full] = cap[full]
    node_num = node_num.astype(np.uint32)
    big = node_num > 3
    cores = np.where(big, rng.choice([1, 1, 2, 4, 8], n_jobs), rng.choice([1, 2, 4, 16, 32, 64, 100, 128, 160], n_jobs))
    cpus_raw = cores * 256
    fr = rng.random(n_jobs) < 0.1
    cpus_raw[fr] = rng.choice([64, 128, 384], int(fr.sum()))
    tpn = np.ones(n_jobs, np.uint32)
    tpn_max = tpn.copy()
    gen = (rng.random(n_jobs) < p_general) & (node_num <= 127)
    tpn[gen] = rng.integers(1, 3, int(gen.sum()))
    tpn_max[gen] = tpn[gen] + rng.integers(1, 4, int(gen.sum()))
    ntasks = (node_num * tpn + rng.integers(0, 1 << 30, n_jobs) % (node_num * (tpn_max - tpn) + 1)).astype(np.uint32)
    cpus_raw = np.where(gen, np.minimum(cpus_raw, 4 * 256), cpus_raw)
    gt = np.zeros((n_jobs, 8), np.uint16)
    gs = np.zeros((n_jobs, GRES_ENTRIES), np.uint16)
    for i in range(n_jobs):
        if rng.random() < (0.25 if big[i] else 0.5):
            for e in rng.choice(GRES_ENTRIES, int(rng.integers(1, 3)), replace=False):
                c = int(rng.choice([1, 1, 2, 3, 4, 8, 16])) if not big[i] else 1
                if rng.random() < 0.6:
                    gs[i, e] += c
                    gt[i, names[e]] += c + (int(rng.integers(0, 2)) if rng.random() < 0.3 else 0)
                else:
                    gt[i, names[e]] += c
    mem_task = rng.integers(1, 9, n_jobs).astype(np.uint64) * GiB // 2
    mem_node = np.where(rng.random(n_jobs) < 0.2, rng.integers(0, 4, n_jobs), 0).astype(np.uint64) * GiB
    views = _views(n_jobs, cpus_raw, mem_task, node_num, ntasks, gt, gs, mem_node)
    mand = np.zeros(n_jobs) if fifo else (rng.permutation(n_jobs) + 1) * 997.0 + 0.5
    tl = _log_uniform(rng, 60, 3600 if short else 3 * DAY, n_jobs)
    submit = NOW - 1 - rng.permutation(9 * DAY)[:n_jobs]
    pend = _pending(n_jobs, part, tl, submit, node_num, ntasks, views,
                    rng.choice([1000, 2000, 3000], n_jobs).astype(np.uint32),
                    rng.choice([1000, 2000, 5000], n_jobs).astype(np.uint32),
                    account=rng.integers(0, 6, n_jobs).astype(np.uint32),
                    qos=rng.integers(0, 3, n_jobs).astype(np.uint32),
                    user=rng.integers(0, 20, n_jobs).astype(np.uint32),
                    exclusive=(rng.random(n_jobs) < 0.03).astype(np.uint8), ntpn=(tpn, tpn_max), mandated=mand)
    cfg = Config(priority_type=0 if fifo else 1, scheduled_batch_size=limit or n_jobs, cost_policy=cost_policy,
                 weight_age=500, weight_fair_share=10000, weight_job_size=300,
                 weight_partition=1000, weight_qos=1_000_000, favor_small=bool(seed & 1))
    return cfg, cluster, running, pend, NOW


def overlap_partitions(case, seed, frac=0.4, which=None):
    """The same case with overlapping partitions: every partition (or only those in
    `which`) also lists a share of the previous partition's nodes, so those nodes have
    ONE NodeState seen by two LocalSchedulers (JobScheduler.cpp:5597-5651)."""
    import dataclasses
    cfg, cl, rn, pd, now = case
    rng = np.random.Generator(np.random.PCG64(seed * 31 + 5))
    lists = [cl.part_nodes[cl.part_off[p]:cl.part_off[p + 1]].tolist() for p in range(cl.n_partitions)]
    out = [list(lists[0])]
    for p in range(1, cl.n_partitions):
        prev = lists[p - 1]
        k = int(len(prev) * frac) if which is None or p in which else 0
        extra = rng.choice(prev, k, replace=False).tolist() if k else []
        out.append(sorted(set(lists[p]) | set(extra)))
    off = np.cumsum([0] + [len(x) for x in out]).astype(np.uint32)
    nodes = np.array([n for x in out for n in x], np.uint32)
    cl2 = dataclasses.replace(cl, part_off=off, part_nodes=nodes)
    return cfg, cl2, rn, pd, now


def random_reservations(seed, case, n_resv=4, frac_jobs=0.15, single_node=False):
    """Reservations over a random_case-style case: a mix of expired, active and
    later ones (ResvMeta, Node/NodeDefs.h:81-97); each reserves part of a few
    nodes' resources (whole low cores, some slots). Returns (Reservations,
    pending', running') with a share of the pending jobs submitted into
    reservations (also unknown ones). single_node: one node per reservation — inside
    a reservation the reference orders equal-cost nodes by the addresses of node
    states created in std::unordered_map iteration order (JobScheduler.cpp:5695-5703),
    which no harness controls; one node leaves nothing to order (tests/test_ref_pin.py)."""
    import dataclasses
    from .abi import Reservations
    cfg, cl, rn, pd, now = case
    rng = np.random.Generator(np.random.PCG64(seed * 7919 + 11))
    start, end, off, nodes, res = [], [], [0], [], []
    # a reservation only holds resources that are free: nodes without running
    # allocations, and no node in two live reservations (the reference asserts on
    # over-subscription, PublicHeader.cpp: cpu_count >= rhs.cpu_count)
    busy = np.zeros(cl.n_nodes, bool)
    busy[rn.alloc_node] = True
    pool = [int(x) for x in rng.permutation(np.flatnonzero(~busy))]
    for r in range(n_resv):
        kind = r % 3  # 0 active, 1 later, 2 expired
        if kind == 0:
            st, en = now - int(rng.integers(10, 5000)), now + int(rng.integers(600, 40000))
        elif kind == 1:
            st = now + int(rng.integers(30, 20000)); en = st + int(rng.integers(300, 30000))
        else:
            st, en = now - 9000, now - int(rng.integers(0, 50))
        k = 1 if single_node else min(int(rng.integers(1, max(2, min(6, cl.n_nodes // 3)))), len(pool))
        k = min(k, len(pool))
        mine, pool = pool[:k], pool[k:]
        for n in sorted(mine):
            tot = cl.res_total[n]
            row = np.zeros((), RES_IN_NODE)
            ncores = max(1, int(tot["cpu_raw"]) // 256 // int(rng.integers(2, 5)))
            row["cpu_raw"] = ncores * 256
            row["mem"] = int(tot["mem"]) // 4
            row["mem_sw"] = int(tot["mem_sw"]) // 4
            left, w = ncores, 0
            core = np.zeros(CORE_WORDS, np.uint64)
            while left > 0 and w < CORE_WORDS:
                take = min(left, 64)
                core[w] = np.uint64((1 << take) - 1) & tot["core"][w]
                left -= take; w += 1
            row["core"] = core
            row["gres"] = tot["gres"] & np.uint16(0x3)  # the two lowest slots of every entry
            nodes.append(n); res.append(row)
        off.append(len(nodes)); start.append(st); end.append(en)
    resv = Reservations(start, end, off, np.array(nodes, np.uint32), np.array(res, RES_IN_NODE))
    pr = np.full(pd.n, 0xFFFFFFFF, np.uint32)
    pick = rng.random(pd.n) < frac_jobs
    pr[pick] = rng.integers(0, n_resv + 1, int(pick.sum())).astype(np.uint32)  # n_resv = an unknown reservation
    pd2 = dataclasses.replace(pd, reservation=pr)
    # running jobs: the cluster's own, plus one job inside every reservation that has
    # started (one reserved core and 1 GiB on the reservation's first node)
    cols = {f: getattr(rn, f) for f in rn.__dataclass_fields__ if f != "reservation"}
    rr = [0xFFFFFFFF] * rn.n
    extra = []
    for r in range(n_resv):
        if start[r] <= now < end[r] and off[r + 1] > off[r]:
            row = np.zeros((), RES_IN_NODE)
            src = res[off[r]]
            low = int(src["core"][0]) & -int(src["core"][0])
            row["cpu_raw"] = 256; row["mem"] = GiB; row["mem_sw"] = GiB
            core = np.zeros(CORE_WORDS, np.uint64); core[0] = np.uint64(low); row["core"] = core
            extra.append((r, nodes[off[r]], row))
    if extra:
        k = len(extra)
        ap = lambda a, v, dt: np.concatenate([a, np.array(v, dt)])
        cols["start_time"] = ap(rn.start_time, [now - 100] * k, np.int64)
        cols["end_time"] = ap(rn.end_time, [now + 777 + 13 * i for i in range(k)], np.int64)
        cols["node_num"] = ap(rn.node_num, [1] * k, np.uint32)
        cols["partition_priority"] = ap(rn.partition_priority, [1000] * k, np.uint32)
        cols["qos_priority"] = ap(rn.qos_priority, [1000] * k, np.uint32)
        cols["account"] = ap(rn.account, [0] * k, np.uint32)
        cols["view_cpu_raw"] = ap(rn.view_cpu_raw, [256] * k, np.int64)
        cols["view_mem"] = ap(rn.view_mem, [GiB] * k, np.uint64)
        cols["alloc_off"] = np.concatenate([rn.alloc_off, rn.alloc_off[-1] + 1 + np.arange(k, dtype=np.uint32)])
        cols["alloc_node"] = ap(rn.alloc_node, [e[1] for e in extra], np.uint32)
        cols["alloc_res"] = np.concatenate([rn.alloc_res, np.array([e[2] for e in extra], RES_IN_NODE)])
        rr += [e[0] for e in extra]
    from .abi import Running
    rn2 = Running(**cols, reservation=np.array(rr, np.uint32))
    return resv, pd2, rn2


def random_qos(seed, cluster, pend, tight=1.0, n_parents=4, invalid_frac=0.1):
    """QoS limits + account chains + (partly pre-filled) usage for a pending table
    (config 3's QoS filter, SURVEY.md §8a R12). Accounts 0..A-1 are the leaves the
    jobs name; each has a parent A + a % n_parents and all share the root; a
    job's chain is [leaf, parent, root]. `tight` scales the limits: ~1 makes every
    reason code occur, large values let everything through."""
    from .abi import META_RESOURCE, TRES_LIMIT, QosTable

    rng = np.random.default_rng(1000 + seed)
    n = pend.n
    n_qos = int(pend.qos.max()) + 1 if n else 1
    n_users = int(pend.user.max()) + 1 if n else 1
    leaves = int(pend.account.max()) + 1 if n else 1
    n_accounts = leaves + n_parents + 1
    chain_off = (np.arange(n + 1, dtype=np.uint32) * 3).astype(np.uint32)
    chain = np.empty((n, 3), np.uint32)
    chain[:, 0] = pend.account
    chain[:, 1] = leaves + pend.account % n_parents
    chain[:, 2] = leaves + n_parents
    # some jobs with a shorter / empty chain
    short = rng.random(n) < 0.1
    lens = np.where(short, rng.integers(0, 3, n), 3).astype(np.uint32)
    chain_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
    chain_acct = np.concatenate([chain[i, :lens[i]] for i in range(n)]) if n else np.zeros(0, np.uint32)
    per_q = max(1, n // n_qos)
    big = np.iinfo(np.int64).max // 4

    def lim(scale_cpu, scale_gres):
        t = np.zeros(n_qos, TRES_LIMIT)
        t["view"]["cpu_raw"] = np.where(rng.random(n_qos) < 0.3, big, (rng.integers(8, 64, n_qos) * 256 * scale_cpu * tight).astype(np.int64))
        t["view"]["mem"] = np.where(rng.random(n_qos) < 0.3, np.uint64(1) << np.uint64(62),
                                    (rng.integers(32, 256, n_qos) * scale_cpu * tight).astype(np.uint64) << np.uint64(30))
        t["view"]["mem_sw"] = 0
        t["gres_name_present"] = rng.integers(0, 4, n_qos)
        t["gres_spec_present"] = rng.integers(0, 1 << max(cluster.n_gres_entries, 1), n_qos)
        t["view"]["gres_total"] = np.minimum(65535, rng.integers(1, 16, (n_qos, 8)) * scale_gres * tight).astype(np.uint16)
        t["view"]["gres_spec"] = np.minimum(65535, rng.integers(1, 12, (n_qos, GRES_ENTRIES)) * scale_gres * tight).astype(np.uint16)
        return t

    q = QosTable(
        n_users=n_users, n_accounts=n_accounts,
        valid=(rng.random(n_qos) >= invalid_frac).astype(np.uint8),
        max_jobs_per_user=np.minimum(2**31, rng.integers(1, 6, n_qos) * tight).astype(np.uint32),
        max_jobs_per_account=np.minimum(2**31, rng.integers(4, 24, n_qos) * tight).astype(np.uint32),
        max_jobs=np.minimum(2**31, rng.integers(per_q // 8 + 1, per_q + 2, n_qos) * tight).astype(np.uint32),
        max_cpus_per_user_raw=np.minimum(big, rng.integers(16, 128, n_qos) * 256 * tight).astype(np.int64),
        max_wall=np.where(rng.random(n_qos) < 0.4, 0, (rng.integers(4, 64, n_qos) * 3600 * tight)).astype(np.int64),
        max_tres_per_user=lim(1, 1), max_tres_per_account=lim(4, 3), max_tres=lim(16, 8),
        chain_off=chain_off, chain_acct=chain_acct,
    )
    # usage left behind by jobs that are already running
    for arr, p in ((q.user_usage, 0.15), (q.account_usage, 0.3), (q.qos_usage, 0.5)):
        m = rng.random(len(arr)) < p
        k = int(m.sum())
        arr["cpu_raw"][m] = rng.integers(0, 16, k) * 256
        arr["mem"][m] = rng.integers(0, 32, k).astype(np.uint64) << np.uint64(30)
        arr["jobs_count"][m] = rng.integers(0, 3, k)
        arr["wall_time"][m] = rng.integers(0, 7200, k)
        for e in range(cluster.n_gres_entries):
            c = rng.integers(0, 3, k).astype(np.uint32)
            arr["gres_spec"][m, e] = c
            arr["gres_total"][m, cluster.gres_entry_name[e]] += c
    return q


CONFIGS = {1: config1, 2: config2, 3: config3, 4: config4, 5: config5}


# ---------------------------------------------------------------------------
# Steps of running jobs (JobInCtld::SchedulePendingSteps): the jobs a NodeSelect
# pass starts now become running jobs whose step_res_avail_ is their allocation
# (JobScheduler.cpp:1277), each with a FIFO queue of srun / crun steps.
# ---------------------------------------------------------------------------
def started_jobs(pending: Pending, placements) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(node_off, node, avail) of the jobs `placements` starts now, in job-id order."""
    started = np.flatnonzero(placements.reason == 0)
    nn = pending.node_num[started].astype(np.int64)
    node_off = np.zeros(len(started) + 1, np.uint32)
    node_off[1:] = np.cumsum(nn)
    rows = (np.repeat(placements.alloc_off[started].astype(np.int64), nn)
            + np.arange(int(nn.sum())) - np.repeat(node_off[:-1].astype(np.int64), nn))
    return node_off, placements.alloc_node[rows].copy(), placements.alloc_res[rows].copy()


def _step_ntpn(ntasks, nn, umin, umax):
    """AcquireStepAttributes' ntasks_per_node bounds (JobScheduler.cpp:6410-6424)."""
    dist_max = ntasks - nn + 1
    tmax = dist_max if umax == 0 else min(umax, dist_max)
    tmin = max(umin, ntasks - (nn - 1) * tmax, 1)
    tmax = min(tmax, ntasks - (nn - 1) * tmin)
    return tmin, tmax


def step_case(seed, select, base=None, max_steps=6, one_type_per_name=False, **case_kw):
    """(cluster, StepJobs, Steps) drawn over the jobs a NodeSelect case starts now.

    select(cfg, cluster, running, pending, now) -> Placements runs the NodeSelect pass
    (the GPU path or a CPU restatement); base is that case (default: random_case(seed,
    ntpn_range=True, one_type_per_name=..., **case_kw)). Every job gets 0..max_steps
    FIFO steps: ntasks_per_node ranges, include / exclude lists (with unknown hosts and
    nodes outside the job), fractional and integer cpus, typed and untyped gres on the
    node or the task request, steps that take the whole allocation, steps that cannot
    fit (so later steps that would fit stay pending), and homogeneous requests whose
    equal task counts tie in the heap."""
    from .abi import StepJobs
    if base is None:
        base = random_case(seed, ntpn_range=True, one_type_per_name=one_type_per_name, **case_kw)
    cfg, cluster, running, pending, now = base
    node_off, node, avail = started_jobs(pending, select(cfg, cluster, running, pending, now))
    rng = np.random.Generator(np.random.PCG64(seed ^ 0x57E9))
    n_jobs = len(node_off) - 1
    n_steps = rng.integers(0, max_steps + 1, n_jobs)
    draw = _StepDraw(cluster)
    for j in range(n_jobs):
        draw.job(rng, node[node_off[j]:node_off[j + 1]], avail[node_off[j]:node_off[j + 1]], int(n_steps[j]))
    jobs = StepJobs(node_off, node, avail, np.array(draw.step_off, np.uint32))
    return cluster, jobs, draw.steps()


class _StepDraw:
    """The step draw of step_case: steps appended job by job (`job` draws `n` steps for a
    job with nodes `node` and avail rows `a`), as one Steps table."""

    def __init__(self, cluster):
        self.cluster = cluster
        self.names = np.array(list(cluster.gres_entry_name) + [0] * (GRES_ENTRIES - cluster.n_gres_entries))
        self.cols = {k: [] for k in ("node_num", "ntasks", "tmin", "tmax")}
        self.req_node, self.req_task, self.incl, self.excl = [], [], [[0], []], [[0], []]
        self.step_off = [0]

    def job(self, rng, node, a, n):
        cluster, names, incl, excl = self.cluster, self.names, self.incl, self.excl
        nk = len(node)
        cpu_min, mem_min = int(a["cpu_raw"].min()), int(a["mem"].min())
        gres_any = np.bitwise_or.reduce(a["gres"], axis=0) if nk else np.zeros(GRES_ENTRIES, np.uint16)
        ents = [e for e in range(cluster.n_gres_entries) if gres_any[e]]
        for _ in range(n):
            vn, vt = np.zeros((), RES_VIEW), np.zeros((), RES_VIEW)
            kind = rng.random()
            if kind < 0.12:  # the whole allocation: one task per node, everything the smallest node holds
                nn, ntasks, tmin, tmax = nk, nk, 1, 1
                vt["cpu_raw"], vt["mem"], vt["mem_sw"] = cpu_min, mem_min, mem_min
                for e in ents:
                    cnt = min(bin(int(x)).count("1") for x in a["gres"][:, e])
                    if cnt:
                        vt["gres_spec"][e] = cnt
                        vt["gres_total"][names[e]] += cnt
            elif kind < 0.22:  # does not fit: blocks this job's queue
                nn = min(nk + int(rng.integers(0, 2)), 127)
                ntasks, tmin, tmax = nn, 1, 1
                vt["cpu_raw"] = cpu_min + 256 if nn == nk else 64
            else:
                nn = int(rng.integers(1, nk + 1))
                ntasks = nn * int(rng.choice([1, 1, 2, 3]))
                if rng.random() < 0.5:
                    ntasks += int(rng.integers(0, nn + 1))
                tmin, tmax = _step_ntpn(ntasks, nn, int(rng.choice([1, 1, 2])), int(rng.choice([0, 0, 1, 2, 4])))
                if tmin > tmax:
                    ntasks, tmin, tmax = nn, 1, 1
                vt["cpu_raw"] = int(rng.choice([64, 128, 384, 256, 256, 512, 1024]))
                mem = int(rng.choice([0, 256 << 20, 1 << 30]))
                vt["mem"], vt["mem_sw"] = mem, mem
                if rng.random() < 0.2:
                    vn["mem"] = vn["mem_sw"] = int(rng.choice([256 << 20, 1 << 30]))
                if ents and rng.random() < 0.35:
                    e = int(rng.choice(ents))
                    v = vn if rng.random() < 0.5 else vt
                    v["gres_total"][names[e]] += 1
                    if rng.random() < 0.5:
                        v["gres_spec"][e] += 1
            if rng.random() < 0.12:  # include list: a subset of the job's nodes, maybe an unknown host / outsider
                sub = sorted(rng.choice(node, int(rng.integers(1, nk + 1)), replace=False).tolist())
                if rng.random() < 0.3:
                    sub.append(0xFFFFFFFF if rng.random() < 0.5 else int(rng.integers(0, cluster.n_nodes)))
                incl[1] += sub
            incl[0].append(len(incl[1]))
            if rng.random() < 0.12:
                excl[1] += sorted(rng.choice(node, int(rng.integers(1, nk + 1)), replace=False).tolist())
            excl[0].append(len(excl[1]))
            for k, v in zip(self.cols, (nn, ntasks, tmin, tmax)):
                self.cols[k].append(v)
            self.req_node.append(vn)
            self.req_task.append(vt)
        self.step_off.append(len(self.cols["node_num"]))

    def steps(self):
        from .abi import Steps
        c, incl, excl = self.cols, self.incl, self.excl
        return Steps(c["node_num"], c["ntasks"], c["tmin"], c["tmax"],
                     np.array(self.req_node, RES_VIEW).reshape(-1), np.array(self.req_task, RES_VIEW).reshape(-1),
                     np.array(incl[0], np.uint32), np.array(incl[1], np.uint32),
                     np.array(excl[0], np.uint32), np.array(excl[1], np.uint32))


def step_pass_stream(seed, node_off, node, avail, job_ids, cluster, max_steps=3, p_job=0.3):
    """Step arrivals of one pass of the step scheduler over the jobs `job_ids` (indices
    into the CSR node_off / node / avail: a job's nodes and its allocation, which sizes
    its steps as in step_case): each job gets 1..max_steps new steps with probability
    p_job, drawn by step_case's draw. Returns (job index of each new step, Steps)."""
    rng = np.random.Generator(np.random.PCG64(seed ^ 0x5A55))
    draw = _StepDraw(cluster)
    owner = []
    for j in job_ids:
        if rng.random() >= p_job:
            continue
        n = int(rng.integers(1, max_steps + 1))
        draw.job(rng, node[node_off[j]:node_off[j + 1]], avail[node_off[j]:node_off[j + 1]], n)
        owner += [int(j)] * n
    return np.array(owner, np.int64), draw.steps()
