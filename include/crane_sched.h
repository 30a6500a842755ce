/*
 * crane_sched.h — C-ABI of the H100-native CraneCtld scheduling hot path.
 *
 * This is the drop-in boundary for ONE call in the reference daemon:
 *
 *     m_node_selection_algo_->NodeSelect(now, running_jobs, pending_jobs);
 *         -- /root/reference/src/CraneCtld/JobScheduler.cpp:1141
 *         -- declared at src/CraneCtld/JobScheduler.h:254-257
 *
 * The reference has no FFI for this path (it is an in-process C++ virtual
 * interface, SURVEY.md §8b); the entry points below are what a cgo/FFI-free
 * C++ caller (the NodeSelect-shaped adaptor in cranesched_b200/adaptor/) binds.
 * Everything is plain-old-data: pointers + sizes, no C++/torch types.
 *
 * Conventions
 *   - times are int64 unix seconds (the reference truncates `now` to 1 s,
 *     JobScheduler.cpp:1071); "unset" start/end time is 0.
 *   - cpu amounts are the raw value of the reference's
 *     cpu_t = fpm::fixed<int64_t,__int128,8> (PublicHeader.h:44): cpus * 256.
 *   - nodes, partitions, accounts, qos, users are dense indices. Node index
 *     order is the documented tie-break for equal-cost nodes (the reference
 *     uses heap-pointer order, JobScheduler.h:588).
 *   - sets of core ids / gres slot ids (std::set in the reference,
 *     PublicHeader.h:412-479,540-558) are bit masks: core bit i = core id i;
 *     slot bit i of gres entry e = the i-th slot (lexicographic slot-path
 *     order) of that (name,type) on that node.
 *   - every `*_off` input array is a CSR offsets array of n+1 entries that
 *     starts at 0 and never decreases; anything else is CRANE_EINVAL.
 *   - all functions return 0 on success or a negative CRANE_E* code; they
 *     never throw and never fall back to a CPU implementation.
 */
#ifndef CRANE_SCHED_H_
#define CRANE_SCHED_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CRANE_CORE_WORDS 4   /* <= 256 cores per node                       */
#define CRANE_GRES_ENTRIES 8 /* (name,type) dictionary entries, cluster-wide */
#define CRANE_GRES_NAMES 8   /* distinct gres names                          */
#define CRANE_MAX_SLOTS 16   /* slots per (name,type) per node               */

/* error codes */
#define CRANE_OK 0
#define CRANE_EINVAL (-22)   /* malformed input (see crane_sched_last_error)  */
#define CRANE_ENOMEM (-12)
#define CRANE_ENODEV (-19)   /* no CUDA device / kernel image not loadable    */
#define CRANE_ECUDA (-5)     /* CUDA runtime error during the call            */
#define CRANE_ENOSYS (-38)   /* feature outside the built scope (see DESIGN)  */

/* Mirrors ResourceInNodeV3 (PublicHeader.h:562-615): concrete per-node
 * resources. 72 bytes. */
typedef struct crane_res_in_node {
  int64_t cpu_raw;                    /* CpuSet::cpu_count raw               */
  uint64_t mem;                       /* bytes                               */
  uint64_t mem_sw;                    /* bytes                               */
  uint64_t core[CRANE_CORE_WORDS];    /* CpuSet::core_ids                    */
  uint16_t gres[CRANE_GRES_ENTRIES];  /* slot masks per dictionary entry     */
} crane_res_in_node_t;

/* Mirrors ResourceView (PublicHeader.h:671-737): counts only. 56 bytes.
 * gres_total[g] = GresCount::total of name g; gres_spec[e] =
 * GresCount::specified[type of entry e]. A name with total==0 and no
 * specified count is "not requested". */
typedef struct crane_res_view {
  int64_t cpu_raw;
  uint64_t mem;
  uint64_t mem_sw;
  uint16_t gres_total[CRANE_GRES_NAMES];
  uint16_t gres_spec[CRANE_GRES_ENTRIES];
} crane_res_view_t;

/* Scheduler knobs: Config::Priority (CtldPublicDefs.h:151-163),
 * ScheduledBatchSize (:231), and the constants at JobScheduler.h:262-264. */
typedef struct crane_sched_config {
  uint32_t priority_type; /* 0 = BasicPriority (JS.h:177), 1 = MultiFactor   */
  uint32_t favor_small;
  uint64_t max_age_s;
  uint32_t weight_age;
  uint32_t weight_fair_share;
  uint32_t weight_job_size;
  uint32_t weight_partition;
  uint32_t weight_qos;
  uint32_t scheduled_batch_size; /* `limit`, JS.cpp:5770                    */
  uint32_t max_jobs_per_node;    /* kAlgoMaxJobNumPerNode (1000)            */
  uint32_t cost_policy;          /* IUpdateNodeCostPolicy (JS.h:30-54): 0 = MinCpuTimeRatioFirst
                                    (the reference's only policy), 1 = BestFit: cost = the node's free
                                    cpu count over all allocations on it, fullest node first — not in
                                    the reference; BASELINE config 4 ("best-fit selection")   */
  int64_t max_time_window_s;     /* kAlgoMaxTimeWindow (7 d)                */
} crane_sched_config_t;

/* Node table + partition membership: what NodeSelect reads from
 * g_meta_container (JobScheduler.cpp:5597-5651; CranedMeta NodeDefs.h:57-79;
 * PartitionMeta::craned_ids NodeDefs.h:118-121). */
typedef struct crane_cluster {
  uint32_t n_nodes;
  const crane_res_in_node_t* res_total; /* [n_nodes]                          */
  const uint8_t* alive;                 /* [n_nodes]                          */
  const uint8_t* drain;                 /* [n_nodes]                          */
  uint32_t n_partitions;
  const uint32_t* part_off;   /* [n_partitions+1] CSR                         */
  const uint32_t* part_nodes; /* node indices, ascending within a partition   */
  uint32_t n_gres_entries;    /* <= CRANE_GRES_ENTRIES                        */
  uint8_t gres_entry_name[CRANE_GRES_ENTRIES]; /* name id of each entry; the
        entries of one name must be contiguous and names ascending            */
} crane_cluster_t;

/* Mirrors RnJobInScheduler (JobScheduler.h:56-89). */
typedef struct crane_running {
  uint32_t n;
  const int64_t* start_time; /* [n]                                          */
  const int64_t* end_time;   /* [n]                                          */
  const uint32_t* node_num;  /* [n] (the reference reads it uninitialised,
                                JS.cpp:6614; here it is an explicit input)   */
  const uint32_t* partition_priority;
  const uint32_t* qos_priority;
  const uint32_t* account;
  const int64_t* view_cpu_raw; /* allocated_res_view.CpuCount raw            */
  const uint64_t* view_mem;    /* allocated_res_view.GetMemoryBytes          */
  const uint32_t* alloc_off;   /* [n+1] CSR over (node, res) pairs           */
  const uint32_t* alloc_node;
  const crane_res_in_node_t* alloc_res;
  const uint32_t* reservation; /* [n] RnJobInScheduler::reservation as an index into
                                  crane_reservations_t, 0xFFFFFFFF = none; NULL = no job has one */
} crane_running_t;

/* Mirrors the inputs of PdJobInScheduler (JobScheduler.h:91-164). Input order
 * is job-id order (the pending map is a btree, JS.cpp:1092). */
typedef struct crane_pending {
  uint32_t n;
  const uint32_t* partition;     /* partition index; >= n_partitions = none  */
  const int64_t* time_limit;     /* seconds, >= 1                            */
  const int64_t* submit_time;
  const uint32_t* node_num;      /* >= 1                                     */
  const uint32_t* ntasks;
  const uint32_t* ntasks_per_node_min;
  const uint32_t* ntasks_per_node_max;
  const uint8_t* exclusive;
  const uint32_t* partition_priority;
  const uint32_t* qos_priority;
  const uint32_t* account;
  const uint32_t* qos;
  const uint32_t* user;
  const double* mandated_priority;   /* 0.0 = compute (JS.h:158, JS.cpp:6535)*/
  const crane_res_view_t* req_node;  /* req_node_res_view                    */
  const crane_res_view_t* req_task;  /* req_task_res_view                    */
  const crane_res_view_t* req_total; /* req_total_res_view                   */
  const uint32_t* incl_off;  /* [n+1] CSR of included_nodes, or NULL; the index
                                0xFFFFFFFF stands for a host unknown to the cluster */
  const uint32_t* incl_nodes;
  const uint32_t* excl_off;  /* [n+1] CSR of excluded_nodes, or NULL          */
  const uint32_t* excl_nodes;
  const uint32_t* reservation; /* [n] PdJobInScheduler::reservation as an index into
                                  crane_reservations_t, 0xFFFFFFFF = none, an index >= n
                                  = a name the daemon does not know ("Reservation Not
                                  Found"); NULL = no job has one */
} crane_pending_t;

/* Reservations: what NodeSelect reads from g_meta_container->GetResvMetaMapPtr()
 * (JobScheduler.cpp:5655-5713; ResvMeta, Node/NodeDefs.h:81-97). A reservation
 * that has started is an allocation on its nodes until its end and — for the
 * pending jobs submitted into it — a scheduler of its own over node states
 * holding exactly the reserved resources, with the timeline ending at the
 * reservation's end; one that starts later is taken out of its nodes' timelines
 * over [start, end); an expired one (now >= end) is ignored. A job backfilled
 * onto a node whose first reservation starts inside the job's window is
 * labelled "Resource Reserved" (JobScheduler.cpp:5829-5841). */
typedef struct crane_reservations {
  uint32_t n;
  const int64_t* start_time;        /* [n]                                    */
  const int64_t* end_time;          /* [n]                                    */
  const uint32_t* node_off;         /* [n+1] CSR over (node, res) pairs:
                                       ResvMeta::res_total.EachNodeResMap()   */
  const uint32_t* node;             /* node index (a node appears once per reservation) */
  const crane_res_in_node_t* res;   /* resources reserved on that node        */
} crane_reservations_t;

/* pending reasons: the strings NodeSelect writes (JS.cpp:192,5784-5864,6547;
 * docs/en/reference/pending_reason.md:42-54) as codes. */
enum {
  CRANE_REASON_NONE = 0,           /* "" : start now                          */
  CRANE_REASON_PRIORITY = 1,       /* "Priority"                              */
  CRANE_REASON_RESOURCE = 2,       /* "Resource"                              */
  CRANE_REASON_RESERVED = 3,       /* "Resource Reserved"                     */
  CRANE_REASON_PART_NOT_FOUND = 4, /* "Partition Not Found"                   */
  CRANE_REASON_RESV_NOT_FOUND = 5, /* "Reservation Not Found" (JS.cpp:5793)   */
  CRANE_REASON_PREEMPTED = 6,      /* "Preempted" (JS.cpp:5815)               */
  /* written for rows the gate keeps out of the run (JobScheduler.cpp:1090-1113) */
  CRANE_REASON_HELD = 7,             /* "Held"                                */
  CRANE_REASON_BEGIN_TIME = 8,       /* "BeginTime"                           */
  CRANE_REASON_DEPENDENCY = 9,       /* "Dependency"                          */
  CRANE_REASON_DEPENDENCY_NEVER = 10,/* "DependencyNeverSatisfied"            */
  /* written by crane_sched_qos_filter (Accounting/AccountMetaContainer.cpp:382-531) */
  CRANE_REASON_QOS_CPU = 16,       /* "QosCpuResourceLimit"                   */
  CRANE_REASON_QOS_JOBS = 17,      /* "QosJobsResourceLimit"                  */
  CRANE_REASON_QOS_WALL = 18,      /* "QosWallTimeLimit"                      */
  CRANE_REASON_QOS_MEM = 19,       /* "QosMemResourceLimit"                   */
  CRANE_REASON_QOS_GRES = 20,      /* "QosGresResourceLimit"                  */
  CRANE_REASON_QOS_INVALID = 21,   /* "InvalidQOS"                            */
  CRANE_REASON_ERASED = 255,       /* a row removed with crane_sched_pending_erase */
};

/* The fields NodeSelect writes into PdJobInScheduler (JobScheduler.h:116-132).
 * Caller-owned, pre-sized. Job i owns allocation slots
 * [alloc_off[i], alloc_off[i] + node_num[i]) with alloc_off = exclusive prefix
 * sum of pending.node_num (written by the callee). n_alloc[i] is node_num[i]
 * when the job holds a placement (start now, or a backfill reservation) and 0
 * otherwise; slots are ordered by node index ascending. */
typedef struct crane_placements {
  uint8_t* reason;        /* [n]                                             */
  double* priority;       /* [n]                                             */
  int64_t* start_time;    /* [n] 0 = unset                                   */
  int64_t* end_time;      /* [n] 0 = unset                                   */
  uint32_t* n_alloc;      /* [n]                                             */
  uint32_t* alloc_off;    /* [n+1]                                           */
  uint32_t* alloc_node;   /* [sum node_num]                                  */
  uint32_t* alloc_ntasks; /* [sum node_num] craned_id_to_task_num            */
  crane_res_in_node_t* alloc_res; /* [sum node_num] allocated_res            */
} crane_placements_t;

typedef struct crane_sched crane_sched_t; /* opaque handle, one per GPU      */

/* Per-call device timings (CUDA events on the handle's stream), ms. */
typedef struct crane_sched_timing {
  float h2d_ms;
  float init_ms;     /* node state + timeline build (R2,R3,R4)               */
  float priority_ms; /* R5/R6                                                */
  float feas_ms;     /* capability bitmap (R7 predicate ⊕ R8)                */
  float commit_ms;   /* sequential select/backfill/update (R7,R9,R10)        */
  float d2h_ms;
  float total_ms;
  uint32_t kernel_launches;
  float qos_ms;      /* device time of the last crane_sched_qos_filter (R12)     */
} crane_sched_timing_t;

/* ---- lifecycle ---------------------------------------------------------- */
/* Replaces: construction of SchedulerAlgo + IPrioritySorter
 * (JobScheduler.cpp:111-121). device = CUDA ordinal. */
int crane_sched_create(const crane_sched_config_t* cfg, int device,
                       crane_sched_t** out);
void crane_sched_destroy(crane_sched_t* h);
const char* crane_sched_last_error(const crane_sched_t* h);

/* Replaces: the node/partition snapshot NodeSelect takes from
 * g_meta_container every tick (JobScheduler.cpp:5603-5651). Call when the node
 * set, alive/drain flags or partition membership change.
 * A node may be listed by several partitions: it then has ONE state shared by
 * their LocalSchedulers (JobScheduler.cpp:5622), and every connected group of
 * such partitions is scheduled as one unit, job by job in priority order, each
 * job in its own partition's node order (at most 8 partitions per group, else
 * CRANE_ENOSYS). Partitions that share nothing keep their independent loops. */
int crane_sched_set_cluster(crane_sched_t* h, const crane_cluster_t* cluster);

/* Replaces: the reservation snapshot of NodeSelect (JobScheduler.cpp:5655-5713).
 * Call after crane_sched_set_cluster (which clears the reservations) whenever
 * the reservation set changes; resv == NULL or n == 0 = none. */
int crane_sched_set_reservations(crane_sched_t* h, const crane_reservations_t* resv);

/* ---- the hot path -------------------------------------------------------- */
/* Replaces: SchedulerAlgo::NodeSelect (JobScheduler.cpp:5543-5868), host
 * buffers in, host buffers out; blocking; single caller thread. */
int crane_sched_node_select(crane_sched_t* h, int64_t now,
                            const crane_running_t* running,
                            const crane_pending_t* pending,
                            crane_placements_t* out);

/* The same call split at the PCIe boundary, for callers that keep the pending
 * table resident (SURVEY.md §8f rank 1) and for measurement:
 *   upload  = H2D of running+pending tables (async on the handle's stream)
 *   run     = every kernel of the tick, device-resident in and out
 *   fetch   = D2H of the placements
 * node_select == upload; run; fetch. */
int crane_sched_upload(crane_sched_t* h, const crane_running_t* running,
                       const crane_pending_t* pending);
int crane_sched_run(crane_sched_t* h, int64_t now);
int crane_sched_fetch(crane_sched_t* h, crane_placements_t* out);

/* The pending table kept resident on the device across ticks (SURVEY.md 8f rank 1):
 * the reference rebuilds its PdJobInScheduler vector from the pending map every
 * tick (JobScheduler.cpp:1090-1113); here a submit appends its row(s)
 * (JobScheduler.cpp:4254), a start or cancel erases its row, and a tick is
 *     crane_sched_set_running(h, running); crane_sched_run(h, now); crane_sched_fetch(h, out)
 * without any H2D of pending jobs. Rows keep their indices (outputs are indexed
 * by row; `out` must be sized for crane_sched_pending_rows(h) rows and the sum of
 * node_num over ALL rows); an erased row reports CRANE_REASON_ERASED and takes
 * part in nothing (priority bounds, batch limit, queue). Rows must arrive in
 * job-id order (equal priorities keep row order). crane_sched_upload ==
 * pending_reset; pending_append; set_running. crane_sched_compact drops the erased rows. */
int crane_sched_pending_reset(crane_sched_t* h);
int crane_sched_pending_append(crane_sched_t* h, const crane_pending_t* rows, uint32_t* first_row);
int crane_sched_pending_erase(crane_sched_t* h, const uint32_t* rows, uint32_t n);
int crane_sched_set_running(crane_sched_t* h, const crane_running_t* running);
uint32_t crane_sched_pending_rows(const crane_sched_t* h);

/* The running table kept resident on the device across ticks. Rows keep their
 * index until the table is replaced; an erased row is a tombstone that takes part
 * in nothing (timelines, initial cost, priority bounds, fair-share service).
 * A steady-state tick is
 *     crane_sched_start(h, started, n, &first);    after the previous run
 *     crane_sched_running_erase(h, ended, m);
 *     crane_sched_keep_running(h, NULL); crane_sched_run(h, now); crane_sched_fetch(h, out)
 * and uploads no job data. crane_sched_set_running == reset; running_append;
 * keep_running; crane_sched_compact drops the tombstones in place. Reservation
 * indices of running rows follow crane_sched_set_reservations, as for pending rows.
 *
 * running_append: appends host rows (recovery at daemon start, jobs started
 *   elsewhere), checked as set_running checks them; *first_row (optional) = the
 *   index of the first new row.
 * running_erase: a job ended or was cancelled (CranedMetaContainer FreeResourceFromNode).
 * start: moves the given pending rows into the running table on the device, from
 *   the last run's placements (JobScheduler.cpp:1273-1305): start / end time from the
 *   placement; node_num, partition_priority, qos_priority, account and reservation
 *   from the pending row; the allocation rows are the job's placement rows; the
 *   view is their sum. New rows follow the order of `pending_rows`; the pending rows
 *   are then erased. CRANE_EINVAL for a row out of range, erased, listed twice, or
 *   whose reason after the last run (and any crane_sched_qos_filter) is not
 *   CRANE_REASON_NONE. Needs a completed run and voids its outputs. CRANE_ENOSYS on a
 *   sharded handle (set_shard n_ranks > 1).
 * keep_running: the next run uses the running table as it stands on the device.
 *   Builds the run's view of the live rows (regrouped only when the rows or the
 *   cluster / reservation layout changed) and sizes the work buffers for the current
 *   pending table; then crane_sched_run may be called. Allocations on nodes outside
 *   the node states are ignored (JobScheduler.cpp:5719); a node index >= n_nodes is
 *   CRANE_EINVAL. *device_ms (optional) receives the CUDA-event time of its kernels. */
int crane_sched_running_append(crane_sched_t* h, const crane_running_t* rows, uint32_t* first_row);
int crane_sched_running_erase(crane_sched_t* h, const uint32_t* rows, uint32_t n);
int crane_sched_start(crane_sched_t* h, const uint32_t* pending_rows, uint32_t n, uint32_t* first_row);
int crane_sched_keep_running(crane_sched_t* h, float* device_ms);
uint32_t crane_sched_running_rows(const crane_sched_t* h);

/* ---- the gate of the resident pending table ----------------------------------- */
/* Before NodeSelect the daemon leaves out of the pending vector every job that is held,
 * whose begin time is still ahead, or whose dependencies are not met
 * (JobScheduler.cpp:1090-1113). Such rows stay in the resident table: each run
 * (crane_sched_run) first evaluates, per row and in this order,
 *     held                                    -> CRANE_REASON_HELD
 *     begin_time > now                        -> CRANE_REASON_BEGIN_TIME
 *     dependencies not met (is_met(now))      -> CRANE_REASON_DEPENDENCY_NEVER if they
 *                                                can never be met (is_failed), else
 *                                                CRANE_REASON_DEPENDENCY
 * and a gated row takes part in nothing, exactly as an erased row: not in the priority
 * bounds, the fair-share account set, the batch limit or the queue. It reports its
 * reason, start / end time 0, n_alloc 0 and zero allocation rows; its priority is
 * unspecified (the daemon does not write it). The dependency state of a row is
 * DependenciesInJob (CtldPublicDefs.h:413-428): entries not yet resolved, is_or and
 * ready_time; an event of a dependee sets ready_time = is_or ? min(ready_time, t + delay)
 * : max(ready_time, t + delay) and resolves the entry;
 *     is_met(now) = (is_or || no entry left) && ready_time <= now
 *     is_failed   = ready_time == CRANE_TIME_FUTURE && (!is_or || no entry left).
 * Times: CRANE_TIME_PAST / CRANE_TIME_FUTURE stand for absl::InfinitePast / InfiniteFuture;
 * t + delay saturates as absl does (an infinite t stays infinite, a finite sum beyond the
 * int64 range is CRANE_TIME_FUTURE). Event times (cancel, end, begin) are whole seconds:
 * the daemon's own carry sub-second parts while its `now` is truncated (JobScheduler.cpp:
 * 1071), so round them UP to the next second. That keeps is_met / is_failed exactly as the
 * daemon computes them, because min, max and + whole-second delays commute with ceil;
 * truncating could let a dependent pass one tick early. A table on which no gate call was
 * made since crane_sched_pending_reset (which clears all gate state) runs exactly as
 * before. On a sharded handle every rank must issue the same gate calls, as it does
 * uploads. Every call here needs set_cluster and voids the last run, like pending_erase. */
#define CRANE_TIME_PAST INT64_MIN
#define CRANE_TIME_FUTURE INT64_MAX

/* DependencyType (PublicDefs.proto:136-141) */
enum { CRANE_DEP_AFTER = 0, CRANE_DEP_AFTER_ANY = 1, CRANE_DEP_AFTER_OK = 2, CRANE_DEP_AFTER_NOT_OK = 3 };
/* What a dependency entry waits on */
enum {
  CRANE_DEPENDEE_PENDING = 0, /* a pending row of this table                            */
  CRANE_DEPENDEE_RUNNING = 1, /* a running row: AFTER resolves at once at its start time */
  CRANE_DEPENDEE_EVENT = 2,   /* already resolved at event_time (recovery from the DB,
                                 re-sending a row's state after compaction: one EVENT
                                 entry at the row's ready_time reproduces it)           */
};

/* The dependency lists of pending rows (JobInCtld::SetDependency and AddDependent at
 * submit, CtldPublicDefs.cpp:1600-1626; JobScheduler.cpp:4215-4248). Row k of the call is
 * pending row row[k]; its entries are [dep_off[k], dep_off[k+1]). */
typedef struct crane_dependencies {
  uint32_t n;
  const uint32_t* row;        /* [n] pending rows                                    */
  const uint8_t* is_or;       /* [n] Dependencies::is_or                            */
  const uint32_t* dep_off;    /* [n+1] CSR over the entries                          */
  const uint8_t* kind;        /* CRANE_DEPENDEE_*                                    */
  const uint32_t* dependee;   /* pending or running row (ignored for EVENT)          */
  const uint8_t* type;        /* CRANE_DEP_*                                         */
  const uint64_t* delay_s;    /* < 2^62                                              */
  const int64_t* event_time;  /* EVENT entries; NULL when the call has none          */
} crane_dependencies_t;

/* set_gate: hold flag and begin time of resident rows (SetHeld, HoldReleaseJobAsync, a
 *   begin-time change, submit); `held` or `begin_time` NULL = unchanged. A row that never
 *   had one is not held and begins at CRANE_TIME_PAST.
 * pending_depend: gives rows their dependency list. CRANE_EINVAL when a row is out of
 *   range, erased, listed twice or already has a list, when a dependee row is out of
 *   range, erased or ended (the daemon's missing-dependency rejection) or is the row
 *   itself, when one row lists the same dependee twice, or for a type > 3, a kind > 2 or
 *   a delay >= 2^62. A RUNNING dependee resolves an AFTER entry at once at its start time.
 * pending_cancel: pending_erase of cancelled jobs, and their events (JobScheduler.cpp:
 *   4067-4073): AFTER and AFTER_ANY at cancel_time, AFTER_OK and AFTER_NOT_OK at
 *   CRANE_TIME_FUTURE.
 * running_end: running_erase of ended jobs, and their events (JobScheduler.cpp:4531-4538)
 *   at end_time[k] (the daemon's recorded end time): AFTER_ANY; AFTER_OK if exit_code[k]
 *   == 0, else at CRANE_TIME_FUTURE; AFTER_NOT_OK the other way round.
 * crane_sched_start also resolves the AFTER entries on the started rows at their
 *   placement's start time (JobScheduler.cpp:1549); their other entries follow the job to
 *   its new running row.
 * pending_erase and running_erase fire nothing: a row with dependents leaves through
 * pending_cancel or running_end. crane_sched_set_running replaces the running table, so
 * entries waiting on running rows must be re-sent (pending_reset, pending_append,
 * set_gate, pending_depend with EVENT entries for what was resolved) when it is used to
 * compact a table with dependencies; crane_sched_compact compacts with the dependency
 * state in place and needs none of that. */
int crane_sched_pending_set_gate(crane_sched_t* h, const uint32_t* rows, uint32_t n, const uint8_t* held,
                                 const int64_t* begin_time);
int crane_sched_pending_depend(crane_sched_t* h, const crane_dependencies_t* deps);
int crane_sched_pending_cancel(crane_sched_t* h, const uint32_t* rows, uint32_t n, int64_t cancel_time);
int crane_sched_running_end(crane_sched_t* h, const uint32_t* rows, uint32_t n, const int64_t* end_time,
                            const uint32_t* exit_code);

/* ---- compaction of the resident tables ------------------------------------------ */
/* Erased rows and resolved dependency entries stay behind in the resident tables, and
 * every run, fetch and dependency event pays for them. crane_sched_compact rewrites the
 * pending and the running table and the dependency entries on the device, keeping only
 * what is live:
 *   pending table  erased rows go; gated rows (held, begin time ahead, dependencies open
 *                  or never satisfiable) are live and stay. Live rows keep their relative
 *                  order: the new index is the row's rank among the live rows, so job-id
 *                  order still holds for later appends. pending_map[old] (pending_rows
 *                  before the call) = the new row, or CRANE_ROW_NONE for an erased row.
 *   running table  the same: running_map[old] (running_rows before the call).
 *   entries        resolved entries and entries of erased rows go. A kept entry's rows
 *                  follow the maps; its gate state (held, begin time, is_or, open entries,
 *                  ready_time) moves with its row. An entry whose dependee row was erased
 *                  without events (pending_erase / running_erase) never fires, before or
 *                  after compaction.
 * Either map may be NULL. Tables without erased rows or resolved entries stay as they are
 * (identity maps); step tables are untouched (they name no pending or running row).
 * Erased rows and resolved entries take part in nothing and the live rows keep their
 * order, so the next run's outputs equal the uncompacted table's, byte for byte, at the
 * mapped rows. Device memory drops to the live rows plus the usual headroom; the peak is
 * the old tables plus the live copy, and CRANE_ENOMEM leaves the tables as they were.
 * No job data crosses PCIe, only the maps. Call it after start / running_end /
 * pending_cancel and before keep_running; it needs set_cluster and voids the last run,
 * like pending_erase (fetch, start and qos_filter need keep_running and run again). On a
 * sharded handle every rank makes the same call. When to compact is the caller's choice. */
#define CRANE_ROW_NONE 0xFFFFFFFFu
int crane_sched_compact(crane_sched_t* h, uint32_t* pending_map, uint32_t* running_map);

/* Blocks until the handle's stream is idle; *run_ms (optional) receives the
 * device time of the last crane_sched_run (CUDA events on that stream). */
int crane_sched_sync(crane_sched_t* h, float* run_ms);

int crane_sched_get_timing(const crane_sched_t* h, crane_sched_timing_t* t);

/* ---- one queue over several GPUs (SURVEY.md 8e) ----------------------------- */
/* The job loop is independent per partition (one LocalScheduler each,
 * JobScheduler.cpp:5757-5766; the reference's "TODO: do it in parallel", :5756):
 * with part_owner[p] == rank this handle commits partition p and leaves every
 * other partition to the handle (GPU) that owns it. Priority, batch limit and
 * queue order are computed from the WHOLE pending table on every rank (upload
 * the same tables everywhere), so they are identical on all ranks. After
 * crane_sched_run the device-side placement columns hold zeros for the jobs this
 * rank does not own (a job without a valid partition belongs to rank 0), which
 * makes the union over ranks a plain sum: one all-reduce(sum) per column of
 * crane_sched_device_placements(), then crane_sched_fetch on any rank returns the
 * whole tick. n_ranks == 1 (the default) switches sharding off. Partitions
 * that share nodes are one unit and must have one owner (CRANE_EINVAL). */
int crane_sched_set_shard(crane_sched_t* h, uint32_t rank, uint32_t n_ranks,
                          const uint32_t* part_owner /* [n_partitions] */);

/* Device pointers of the placement columns of the last crane_sched_run, for the
 * all-reduce above (NCCL through the caller's communicator). `priority` is
 * identical on all ranks and is not part of the exchange. */
typedef struct crane_device_placements {
  void* reason;       /* uint8  [n_jobs]                                      */
  void* start_time;   /* int64  [n_jobs]                                      */
  void* end_time;     /* int64  [n_jobs]                                      */
  void* n_alloc;      /* uint32 [n_jobs]                                      */
  void* alloc_node;   /* uint32 [n_rows]                                      */
  void* alloc_ntasks; /* uint32 [n_rows]                                      */
  void* alloc_res;    /* crane_res_in_node_t [n_rows] = 9 x uint64 per row    */
  uint64_t n_jobs;
  uint64_t n_rows;
} crane_device_placements_t;
int crane_sched_device_placements(crane_sched_t* h, crane_device_placements_t* out);

/* ---- QoS post-filter (R12) ------------------------------------------------ */
/* A ResourceView limit of struct Qos (Account/AccountDefs.h:27-50): max_tres,
 * max_tres_per_user, max_tres_per_account. A gres name / type that is absent
 * from the limit map is "unlimited"; presence is carried by the two masks
 * (bit g = name g present, bit e = dictionary entry e present in `specified`). */
typedef struct crane_tres_limit {
  crane_res_view_t view;
  uint8_t gres_name_present;
  uint8_t gres_spec_present;
  uint8_t pad[6];
} crane_tres_limit_t;

/* MetaResource (Accounting/AccountMetaContainer.h:30-47): running usage of one
 * (user,qos), (account,qos) or qos. */
typedef struct crane_meta_resource {
  int64_t cpu_raw;
  uint64_t mem;
  uint64_t mem_sw;
  uint32_t gres_total[CRANE_GRES_NAMES];
  uint32_t gres_spec[CRANE_GRES_ENTRIES];
  uint32_t jobs_count;
  uint32_t pad;
  int64_t wall_time;
} crane_meta_resource_t;

typedef struct crane_qos_table {
  uint32_t n_qos, n_users, n_accounts;
  /* limits, indexed by qos id (struct Qos, AccountDefs.h:27-50) */
  const uint8_t* valid;                 /* 0 -> "InvalidQOS" (deleted / unknown) */
  const uint32_t* max_jobs_per_user;
  const uint32_t* max_jobs_per_account;
  const uint32_t* max_jobs;
  const int64_t* max_cpus_per_user_raw;
  const int64_t* max_wall;              /* seconds; 0 = unlimited               */
  const crane_tres_limit_t* max_tres_per_user;
  const crane_tres_limit_t* max_tres_per_account;
  const crane_tres_limit_t* max_tres;
  /* account chain of every pending job (PdJobInScheduler::account_chain),
   * CSR over account ids, in chain order */
  const uint32_t* chain_off;            /* [n_pending + 1]                      */
  const uint32_t* chain_acct;
  /* usage, read and updated in place (host memory) */
  crane_meta_resource_t* user_usage;    /* [n_users][n_qos]                     */
  crane_meta_resource_t* account_usage; /* [n_accounts][n_qos]                  */
  crane_meta_resource_t* qos_usage;     /* [n_qos]                              */
} crane_qos_table_t;

/* Replaces: the CheckAndMallocQosResource calls of the commit loop
 * (JobScheduler.cpp:1262 -> Accounting/AccountMetaContainer.cpp:164-191, 382-531, 546-587)
 * for the placements of the last crane_sched_run: in job-id (input) order, every
 * job that NodeSelect starts now is checked against its (user,qos), account
 * chain and qos limits and, if it passes, added to the usage; a job that fails
 * gets the QoS reason code (it keeps the timeline reservation it made, as in
 * the reference). `reason` ([n_pending], host) receives the updated reasons.
 * Needs pending.qos and pending.user at upload. CRANE_ENOSYS for an account
 * chain longer than 30, CRANE_EINVAL for an account repeated inside a chain or
 * ids outside the tables. Usage maps are dense here, so the reference's
 * "QosResourceLimit" (entry missing from a map) cannot occur. */
int crane_sched_qos_filter(crane_sched_t* h, const crane_qos_table_t* qos, uint8_t* reason);

/* ---- the step scheduler of running jobs ------------------------------------ */
/* Running jobs with pending steps (srun / crun steps inside an allocation): the
 * job's nodes, its step_res_avail_ (JobInCtld, seeded from the job's allocation
 * at start, JobScheduler.cpp:1277) and its pending_step_ids_ queue. */
typedef struct crane_step_jobs {
  uint32_t n_jobs;
  const uint32_t* node_off;   /* [n_jobs+1] CSR over (job, node) pairs          */
  const uint32_t* node;       /* node index, ascending and distinct in a job    */
  crane_res_in_node_t* avail; /* [node_off[n_jobs]] step_res_avail_ of the job on
                                 that node; read and written in place          */
  const uint32_t* step_off;   /* [n_jobs+1] the job's pending steps, FIFO, are the
                                 rows [step_off[j], step_off[j+1]) of the steps */
} crane_step_jobs_t;

/* The fields of CommonStepInCtld the step scheduler reads, one row per pending
 * step (conventions of crane_pending_t). ntasks_per_node_{min,max} as
 * AcquireStepAttributes leaves them (JobScheduler.cpp:6410-6433). */
typedef struct crane_steps {
  uint32_t n;                        /* == step_off[n_jobs]                      */
  const uint32_t* node_num;          /* 1 .. 127                                 */
  const uint32_t* ntasks;            /* >= node_num                              */
  const uint32_t* ntasks_per_node_min;  /* >= 1                                  */
  const uint32_t* ntasks_per_node_max;
  const crane_res_view_t* req_node;  /* req_node_res_view                        */
  const crane_res_view_t* req_task;  /* req_task_res_view                        */
  const uint32_t* incl_off;  /* [n+1] CSR of included_nodes, or NULL; 0xFFFFFFFF
                                stands for a host unknown to the cluster         */
  const uint32_t* incl_nodes;
  const uint32_t* excl_off;  /* [n+1] CSR of excluded_nodes, or NULL            */
  const uint32_t* excl_nodes;
} crane_steps_t;

/* What SchedulePendingSteps writes. Caller-owned, pre-sized. Step s owns node rows
 * [node_off[s], node_off[s] + node_num[s]) in node-index order (node, tasks on it,
 * its allocated_res: the node allocation plus its task allocations) and task rows
 * [task_off[s], task_off[s] + ntasks[s]) in task-id order (node of the task and
 * task_res_map[task id]); both offsets are exclusive prefix sums written by the
 * callee. Rows of a step that was not scheduled are zero. */
typedef struct crane_step_placements {
  uint32_t* placed;        /* [n_jobs] steps placed at the head of the job's queue */
  uint8_t* scheduled;      /* [n] 1 = scheduled now                             */
  uint32_t* node_off;      /* [n+1]                                             */
  uint32_t* alloc_node;    /* [sum node_num]                                    */
  uint32_t* alloc_ntasks;  /* [sum node_num] craned_task_map[node].size()       */
  crane_res_in_node_t* alloc_res; /* [sum node_num]                             */
  uint32_t* task_off;      /* [n+1]                                             */
  uint32_t* task_node;     /* [sum ntasks]                                      */
  crane_res_in_node_t* task_res;  /* [sum ntasks]                               */
} crane_step_placements_t;

/* Replaces: the JobInCtld::SchedulePendingSteps calls of the step scheduler thread
 * (CtldPublicDefs.cpp:1877-1998; JobScheduler.cpp:1637-1665), for every job at
 * once; blocking. Each job takes its steps in FIFO order; a step that does not fit
 * blocks every later step of its job. Nodes are walked in node-index order (the
 * reference walks an unordered_map). Uses the gres dictionary of
 * crane_sched_set_cluster and no NodeSelect state. *device_ms (optional) receives
 * the CUDA-event time of the step kernel. CRANE_EINVAL for a node out of range or
 * repeated / unordered within a job, node_num == 0, ntasks < node_num or
 * ntasks_per_node_min > _max; CRANE_ENOSYS for node_num > 127 or
 * ntasks_per_node_min == 0. */
int crane_sched_schedule_steps(crane_sched_t* h, const crane_step_jobs_t* jobs,
                               const crane_steps_t* steps, crane_step_placements_t* out,
                               float* device_ms);

/* ---- the step state of running jobs kept resident on the device ------------ */
/* The daemon's step state changes by small events; these calls keep it on the device
 * across passes of the step scheduler thread (JobScheduler.cpp:1637-1665) instead of
 * re-sending every job with pending steps to crane_sched_schedule_steps on every pass.
 * Two tables whose rows keep their index until crane_sched_steps_compact drops their
 * erased rows in place (running steps' allocations included), or until
 * crane_sched_step_jobs_reset empties them (how a caller starts over):
 *   step jobs  one row per running job that can get steps: its nodes (ascending and
 *              distinct) and one step_res_avail_ row per node. Independent of the running
 *              table: set_running, running_erase / running_end, set_cluster and every
 *              NodeSelect call leave it alone.
 *   steps      one row per step, bound to a step-job row, holding its crane_steps_t
 *              columns; pending, scheduled or erased. A scheduled row keeps its node rows
 *              (node, res) on the device so that erasing it gives them back. A job's FIFO
 *              queue is its live pending step rows in row order.
 * Daemon call sites:
 *   job start, SetStepResAvail(allocated_res) (JobScheduler.cpp:1277), batch and calloc
 *     primaries                     step_jobs_start(running rows): copies the running
 *                                   rows' allocation entries into new step-job rows, on
 *                                   the device
 *   crun primary (InitPrimaryStepFromJob takes from avail on the host), a job started
 *     elsewhere, a recovered job    step_jobs_append(host rows; step_off must be NULL)
 *   AddStep (CtldPublicDefs.h:984)  steps_append(steps, job_row[n])
 *   EraseStep (CtldPublicDefs.h:1000) steps_erase: a pending row leaves its queue; a
 *                                   scheduled row's node rows are added back to its
 *                                   job's avail (ResourceInNodeV3 +=)
 *   job leaves m_running_job_map_   step_jobs_erase: the job and all its step rows go,
 *                                   nothing is released
 *   one pass of StepScheduleThread_ steps_run, then steps_fetch
 * Rules:
 *   - every call needs crane_sched_set_cluster (the gres dictionary);
 *   - steps_append gives exactly the CRANE_EINVAL / CRANE_ENOSYS answers
 *     crane_sched_schedule_steps gives for the same step, and CRANE_EINVAL for a job row
 *     out of range or erased;
 *   - step_jobs_start: CRANE_EINVAL for a running row out of range, erased, listed
 *     twice, or whose allocation nodes are not ascending and distinct (rows that
 *     crane_sched_start made always pass; rows of running_append may not, which a flag
 *     on the device reports);
 *   - every erase: CRANE_EINVAL for a row out of range, already erased, listed twice, or
 *     whose job was erased; a refused call changes nothing;
 *   - a pass visits only the jobs that are dirty and have a live pending step. A job
 *     becomes dirty when it is appended or started, gets a step, loses a pending step or
 *     gets an allocation back; every pass clears the flag. This is exact: after a pass
 *     every job with pending steps is blocked at its head, and a job whose avail and
 *     queue did not change would be blocked at the same head again;
 *   - steps_run returns the number of steps it scheduled and of their node and task
 *     rows, which size the caller's buffers; steps_fetch returns only those steps, step
 *     rows ascending, in the layout of crane_step_placements_t (node rows in node-index
 *     order, task rows in task-id order, node_off / task_off prefix sums over the
 *     returned steps). Every later step call voids the fetch;
 *   - no step call changes what NodeSelect reads or writes: the handle's stage (a
 *     crane_sched_start after fetch / qos_filter still works with step calls in
 *     between), the running table's regroup and the pending / running buffers;
 *   - single caller, as every call on the handle: in the daemon both scheduler threads
 *     hold m_running_job_map_mtx_ at their call sites (JobScheduler.cpp:1641).
 * *first (optional) receives the first new row of an append or start; *device_ms
 * (optional) the CUDA-event time of the pass's kernels. */
typedef struct crane_step_results {
  uint32_t* step_row;      /* [n_scheduled] step rows, ascending                       */
  uint32_t* node_off;      /* [n_scheduled+1]                                          */
  uint32_t* alloc_node;    /* [n_node_rows]                                            */
  uint32_t* alloc_ntasks;  /* [n_node_rows]                                            */
  crane_res_in_node_t* alloc_res; /* [n_node_rows]                                     */
  uint32_t* task_off;      /* [n_scheduled+1]                                          */
  uint32_t* task_node;     /* [n_task_rows]                                            */
  crane_res_in_node_t* task_res;  /* [n_task_rows]                                     */
} crane_step_results_t;

int crane_sched_step_jobs_start(crane_sched_t* h, const uint32_t* running_rows, uint32_t n, uint32_t* first);
int crane_sched_step_jobs_append(crane_sched_t* h, const crane_step_jobs_t* jobs, uint32_t* first);
int crane_sched_step_jobs_erase(crane_sched_t* h, const uint32_t* rows, uint32_t n);
int crane_sched_steps_append(crane_sched_t* h, const crane_steps_t* steps, const uint32_t* job_row, uint32_t* first);
int crane_sched_steps_erase(crane_sched_t* h, const uint32_t* rows, uint32_t n);
int crane_sched_steps_run(crane_sched_t* h, uint32_t* n_scheduled, uint32_t* n_node_rows, uint32_t* n_task_rows,
                          float* device_ms);
int crane_sched_steps_fetch(crane_sched_t* h, crane_step_results_t* out);
/* The avail rows of step jobs rows[k], one job after another, into dst (host; NULL =
 * only count them); *n_node_rows (optional) receives their number. */
int crane_sched_step_jobs_avail(crane_sched_t* h, const uint32_t* rows, uint32_t n, crane_res_in_node_t* dst,
                                uint32_t* n_node_rows);
int crane_sched_step_jobs_reset(crane_sched_t* h);
/* Rows of the resident step tables, tombstones included (any pointer may be NULL): step
 * jobs, steps, and node rows of the allocation pool. */
int crane_sched_step_rows(const crane_sched_t* h, uint32_t* step_jobs, uint32_t* steps, uint32_t* alloc_rows);
/* Compaction of the step tables. Erased rows stay behind in both tables, and every
 * scheduled step's node rows stay in the allocation pool even after it ends, so the
 * tables only grow. crane_sched_steps_compact rewrites them on the device, keeping only
 * what is live:
 *   step jobs  rows erased by step_jobs_erase go. step_job_map[old] (step_jobs of
 *              step_rows before the call) = the new row, or CRANE_ROW_NONE. A kept job
 *              keeps its nodes and avail rows byte for byte, its dirty flag and its queue.
 *   steps      erased steps and every step of an erased job go; pending and scheduled
 *              steps stay in their state. step_map[old] likewise.
 *   pool       only the node rows of the scheduled steps that stay, each step pointing at
 *              its new span: a later steps_erase of it gives the same rows back.
 * Kept rows keep their relative order (the new index is the rank among kept rows), so a
 * job's FIFO queue, later appends and every pass's results are unchanged at the mapped
 * rows. Either map may be NULL; with nothing erased the tables stay as they are and the
 * maps are the identity. Needs set_cluster, voids the last steps_fetch as every step call
 * does, and leaves NodeSelect alone (crane_sched_compact and this call touch disjoint
 * tables). Every new buffer is allocated before the first copy, so CRANE_ENOMEM leaves the
 * tables as they were; afterwards device memory holds the kept rows plus the usual
 * headroom. Only row indices cross PCIe, host to device. When to compact is the caller's
 * choice. */
int crane_sched_steps_compact(crane_sched_t* h, uint32_t* step_job_map, uint32_t* step_map);

/* Capability bitmap of the last run (the jobs x nodes feasibility bitmap):
 * bit (rank r, local node q) set iff the r-th job in priority order can run
 * on the q-th node of its partition by total resources and node lists
 * (JobScheduler.cpp:5238-5266). words_per_row = ceil(max_part_size/32).
 * Copies min(cap, rows*words_per_row) words to `dst` (host). For tests. */
int crane_sched_debug_bitmap(crane_sched_t* h, uint32_t* dst, size_t cap_words,
                             uint32_t* rows, uint32_t* words_per_row);

/* Per-partition phase cycle counters of the commit kernel, [n_partitions][16];
 * all zero unless the library was built with -DCRANE_PROFILE (a profiling
 * build, never the shipped one). For tools/. */
int crane_sched_debug_profile(crane_sched_t* h, unsigned long long* dst, size_t cap);

#ifdef __cplusplus
}
#endif
#endif /* CRANE_SCHED_H_ */
