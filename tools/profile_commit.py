"""Phase breakdown of k_commit2 (needs the -DCRANE_PROFILE build)."""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from cranesched_b200 import synth, abi
from cranesched_b200.scheduler import GpuScheduler
from cranesched_b200.build import CSRC

NAMES = ["0 loop top + ring issue", "1 form batch", "2 select", "3 resolve", "4 evaluate", "5 commit", "6 re-key", "7 one-job path",
            "8 #windows of the one-job path", "9 #batches cut: candidates taken (wait)", "10 #batches cut: clash with a re-keyed node", "11 #batches cut: pick failed the exact test",
            "12 #batches cut: backfill without a start", "13 #jobs finished in batches", "14 #batches", "15 #exact tests of the one-job path"]
TIMED = {0, 1, 2, 3, 4, 5, 6, 7}
cfg_id = int(sys.argv[1]) if len(sys.argv) > 1 else 2
kw = {}
if len(sys.argv) > 3:
    kw = dict(n_jobs=int(sys.argv[2]), n_nodes=int(sys.argv[3]))
if os.environ.get("SEED_ID"):
    kw["seed_id"] = int(os.environ["SEED_ID"])
cfg, cl, rn, pd, now = synth.CONFIGS[cfg_id](**kw)
s = GpuScheduler(cfg, 0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "variants", "libcrane_sched_prof.so"))
s.set_cluster(cl)
for _ in range(2):
    out = s.node_select(now, rn, pd)
t = s.timing()
prof = s.debug_profile()
jobs = np.bincount(pd.partition[pd.partition < cl.n_partitions], minlength=cl.n_partitions)
print(json.dumps({k: round(v, 3) for k, v in t.items()}))
crit = max(range(cl.n_partitions), key=lambda p: sum(int(prof[p, i]) for i in TIMED))
for p in range(cl.n_partitions):
    tot = sum(int(prof[p, i]) for i in TIMED)
    nb, nbj = int(prof[p, 14]), int(prof[p, 13])
    print("partition %d: %d jobs, %.0f cycles/job, total %.1f Mcycles%s" % (p, jobs[p], tot / max(jobs[p], 1), tot / 1e6,
                                                                          "  <- critical CTA" if p == crit else ""))
    print("   %-20s %10d batches, %.2f jobs per batch" % ("batches", nb, nbj / max(nb, 1)))
    for i, n in enumerate(NAMES):
        v = int(prof[p, i])
        if i in TIMED:
            print("   %-20s %8.0f cyc/job  %5.1f%%" % (n, v / max(jobs[p], 1), 100.0 * v / max(tot, 1)))
        elif v:
            if i == 12:
                print("   %-20s %10.2f per job" % (n, (v & 0xffffffff) / max(jobs[p], 1)))
                print("   %-20s %10.2f per job" % ("#jobs on the one-job path", (v >> 32) / max(jobs[p], 1)))
            else:
                print("   %-20s %10d  (%.2f per job)" % (n, v, v / max(jobs[p], 1)))
s.close()
