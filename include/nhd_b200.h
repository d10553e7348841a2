/*
 * nhd_b200.h — C-ABI of the H100-native NHD placement solver.
 *
 * This is the drop-in boundary for the one hot path of Viasat/nhd: the node
 * filter -> NUMA/PCIe intersection -> node select -> physical assignment loop.
 * The reference has no FFI; its seam is the Python method surface
 *     Matcher.FindNode(nl, top)                      nhd/Matcher.py:27-63
 *     Node.SetPhysicalIdsFromMapping(mapping, top)   nhd/Node.py:663-841
 *     Node.ClaimPodNICResources(nidx)                nhd/Node.py:644-646
 * driven once per pending pod by NHDScheduler.AttemptScheduling
 * (nhd/NHDScheduler.py:277-304) after NHDScheduler.InitialNodeFilter
 * (nhd/NHDScheduler.py:235-247).  One call of nhd_solve_batch() replaces that
 * whole per-pod sequence for a batch of pods, with the reference's strict
 * sequential semantics (pod i sees the cluster after pods 0..i-1).
 *
 * Conventions: plain C, caller owns every buffer, all functions return an
 * int32 status (0 = NHD_OK, negative = error), no exceptions cross the
 * boundary, a handle is not re-entrant (the reference has a single scheduler
 * thread, nhd/NHDScheduler.py:43).  Every pointer is a HOST pointer unless the
 * name ends in _dev.
 */
#ifndef NHD_B200_H
#define NHD_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- limits of the packed layout (checked by nhd_validate_*) -------------- */
#define NHD_MAX_NUMA           4    /* Node.numa_nodes (== sockets, Node.py:336)      */
#define NHD_MAX_GROUPS         4    /* len(CfgTopology.proc_groups)                   */
#define NHD_MAX_TUPLES         256  /* numa^(groups+1) must not exceed this; numa = the largest NUMA count among the
                                        nodes the filter could accept (active, not in maintenance) at staging time */
#define NHD_MAX_GPUS           16   /* len(Node.gpus)                                 */
#define NHD_MAX_NICS           32   /* len(Node.nics) (schedulable NICs / VFs)        */
#define NHD_MAX_LCORES         256  /* len(Node.cores) (logical cores)                */
#define NHD_MAX_SWITCHES       16   /* distinct PCIe switch ids on one node           */
#define NHD_MAX_SPEED_CLASSES  16   /* distinct NIC link speeds in the cluster        */
#define NHD_MAX_GROUP_GPUS     8    /* len(ProcGroup.group_gpus)                      */
#define NHD_MAX_POD_GPUS       16   /* GPUs requested by one pod                      */
#define NHD_MAX_POD_CORES      72   /* cores requested by one pod                     */
#define NHD_MAX_GROUP_NAMES    64   /* distinct node-group names in the cluster       */

/* ---- return codes ---------------------------------------------------------- */
#define NHD_OK                  0
#define NHD_ERR_INVALID        -1   /* bad argument / malformed record                */
#define NHD_ERR_UNSUPPORTED    -2   /* valid for the reference, outside packed limits */
#define NHD_ERR_CUDA           -3   /* CUDA runtime failure (see nhd_last_error)      */
#define NHD_ERR_NCCL           -4   /* NCCL failure / NCCL not loadable               */
#define NHD_ERR_STATE          -5   /* call order (e.g. solve before load)            */
#define NHD_ERR_LABELS         -6   /* Node.ParseLabels would return False (node ignored) */

/* ---- per-pod outcome (nhd_binding.status) ---------------------------------- */
#define NHD_PLACED              0   /* FindNode found a node and assignment succeeded (NHDScheduler.py:291-304) */
#define NHD_NO_CANDIDATE        1   /* FindNode returned (None,)   (Matcher.py:52,60)                           */
#define NHD_ASSIGN_FAILED       2   /* SetPhysicalIdsFromMapping raised IndexError, clean unwind (Node.py:825-837) */
#define NHD_REF_WOULD_CRASH     3   /* unwind hit the buggy NIC rollback (Node.py:831-835); state as IndexError  */
#define NHD_BAD_MAP_TYPE        4   /* map_type not NUMA/PCI -> (None,) (Matcher.py:45-47)                       */

/* Why a node could not take a NO_CANDIDATE pod (nhd_explain_batch / nhd_explain_pod): the FIRST stage of the
 * reference, in this order, that drops the node, evaluated on the cluster as that pod saw it. */
#define NHD_WHY_GROUP           0   /* no node-group in common with the pod   (NHDScheduler.py:240)          */
#define NHD_WHY_INACTIVE        1   /* node not active                        (NHDScheduler.py:241)          */
#define NHD_WHY_MAINTENANCE     2   /* node in maintenance                    (Matcher.py:73)                */
#define NHD_WHY_HUGEPAGES       3   /* pod's hugepages_gb > node's free        (Matcher.py:78)                */
#define NHD_WHY_BUSY            4   /* GPU pod inside the node's busy window   (Matcher.py:107-111)           */
#define NHD_WHY_GPU             5   /* no NUMA tuple of free GPUs              (Matcher.py:132)               */
#define NHD_WHY_CPU             6   /* no NUMA tuple of free CPU cores         (Matcher.py:214)               */
#define NHD_WHY_NIC             7   /* no NIC combination with the bandwidth   (Matcher.py:270)               */
#define NHD_WHY_INTERSECT       8   /* PCI pruning and/or empty GPU/CPU/NIC intersection (Matcher.py:295-359) */
#define NHD_WHY_COUNT           9
#define NHD_WHY_NONE            0xFF /* nhd_explain_pod: the pod's status is not NHD_NO_CANDIDATE            */

/* CfgTopology.TopologyMapType values (CfgTopology.py:41-45) */
#define NHD_MAP_INVALID         0
#define NHD_MAP_NUMA            1
#define NHD_MAP_PCI             2
#define NHD_MAP_NONE            3

/* nhd_node_rec.flags */
#define NHD_NODE_SMT            0x01  /* Node.smt_enabled   (Node.py:335) */
#define NHD_NODE_ACTIVE         0x02  /* Node.active        (NHDScheduler.py:242) */
#define NHD_NODE_MAINTENANCE    0x04  /* Node.maintenance   (Matcher.py:73) */

/* nhd_pod_group.flags */
#define NHD_GRP_PROC_SMT        0x01  /* ProcGroup.proc_smt   == SMT_ENABLED */
#define NHD_GRP_HELPER_SMT      0x02  /* ProcGroup.helper_smt == SMT_ENABLED */
#define NHD_GRP_HAS_NIC_CORES   0x04  /* any proc core with nic_dir RX or TX (Node.py:742) */

/* nhd_pod.flags */
#define NHD_POD_MISC_SMT        0x01  /* CfgTopology.misc_cores_smt == SMT_ENABLED */

/*
 * nhd_node_rec — the complete decision-relevant state of one Node
 * (nhd/Node.py:100-131), 128 bytes.  Everything the reference reads on the hot
 * path is here; names, MACs, GPU device ids and the NIC speed_used/pods_used
 * counters stay with the caller (they never influence a decision while
 * ENABLE_SHARING is False, Node.py:20,292).
 *
 *  logical core c (Node.cores[c]):  socket(c) = (c % phys_cores) / (phys_cores / n_numa)
 *                                   sibling(c) = c +- phys_cores when SMT      (Node.py:343-350)
 *  gpus[i] / nics[i] are in Node.gpus / Node.nics list order (label order, Node.py:388-432).
 *  A NIC's per-NUMA index NodeNic.idx (Node.py:413-418) is its rank among the
 *  set bits of nic_numa_mask[numa].
 *  Switch ids are node-local 4-bit aliases of NodeGpu/NodeNic.pciesw (only
 *  equality is ever tested: Matcher.py:316-320, Node.py:651).
 */
typedef struct nhd_node_rec {
    uint64_t used[4];            /* bit c = Node.cores[c].used (reserved cores included)      */
    uint16_t gpu_used;           /* bit i = Node.gpus[i].used                                  */
    uint8_t  n_gpus;             /* len(Node.gpus)                                             */
    uint8_t  n_nics;             /* len(Node.nics)                                             */
    uint32_t nic_inuse;          /* bit i = Node.nics[i].pods_used > 0                         */
    int32_t  free_hugepages_gb;  /* Node.mem.free_hugepages_gb                                 */
    uint8_t  n_numa;             /* Node.numa_nodes                                            */
    uint8_t  flags;              /* NHD_NODE_*                                                 */
    uint16_t phys_cores;         /* label nfd-extras-cpu.num_cores (physical cores, Node.py:334) */
    double   busy_time;          /* Node.busy_time (monotonic seconds, Node.py:115,845)        */
    uint64_t group_mask;         /* bit j = cluster group name j in Node.groups                */
    uint16_t gpu_numa_mask[NHD_MAX_NUMA];  /* bit i = (Node.gpus[i].numa_node == k)            */
    uint64_t gpu_sw;             /* nibble i = local switch id of Node.gpus[i]                 */
    uint32_t nic_numa_mask[NHD_MAX_NUMA];  /* bit i = (Node.nics[i].numa_node == k)            */
    uint64_t nic_sw[2];          /* nibble i = local switch id of Node.nics[i]                 */
    uint64_t nic_speed[2];       /* nibble i = speed class of Node.nics[i] (nhd_params.speed_gbps) */
} nhd_node_rec;

/* One ProcGroup of a pod request (CfgTopology.py:82-110), 32 bytes. */
typedef struct nhd_pod_group {
    uint8_t n_gpus;              /* len(group_gpus)                                            */
    uint8_t n_proc;              /* len(proc_cores)                                            */
    uint8_t n_helpers;           /* len(misc_cores) of the group ("helper" cores)              */
    uint8_t flags;               /* NHD_GRP_*                                                  */
    uint8_t gpu_feeders[NHD_MAX_GROUP_GPUS]; /* len(group_gpus[j].cpu_cores)                   */
    uint8_t pad_[4];
    double  rx_gbps;             /* sum of nic_speed over RX proc cores, core order (CfgTopology.py:219-232) */
    double  tx_gbps;             /* same for TX                                                */
} nhd_pod_group;

/* One pending pod: CfgTopology (CfgTopology.py:126-143) + its node-group list
 * (NHDScheduler.py:238, K8SMgr.py:160-163), 144 bytes. */
typedef struct nhd_pod {
    uint8_t  n_groups;           /* len(proc_groups), 1..NHD_MAX_GROUPS                        */
    uint8_t  map_type;           /* NHD_MAP_*                                                  */
    uint8_t  n_misc;             /* len(CfgTopology.misc_cores)                                */
    uint8_t  flags;              /* NHD_POD_*                                                  */
    int32_t  hugepages_gb;       /* CfgTopology.hugepages_gb                                   */
    uint64_t group_mask;         /* bit j = cluster group name j requested by the pod          */
    nhd_pod_group groups[NHD_MAX_GROUPS];
} nhd_pod;

/*
 * nhd_binding — everything AttemptScheduling learns for one pod, 128 bytes:
 * the node, the mapping dict FindNode returns (Matcher.py:452), every value
 * SetPhysicalIdsFromMapping writes into the CfgTopology (Node.py:724-811) and
 * the NIC list handed to ClaimPodNICResources (NHDScheduler.py:302-304).
 */
typedef struct nhd_binding {
    int32_t status;              /* NHD_PLACED ...                                             */
    int32_t node;                /* node index in load order, -1 when none                     */
    uint8_t n_groups;
    uint8_t n_cores;             /* entries used in cores[]                                    */
    uint8_t n_gpus;              /* entries used in gpu_index[]                                */
    uint8_t n_claimed;           /* entries used in claimed_nics[]                             */
    uint8_t gpu_numa[NHD_MAX_GROUPS];      /* mapping['gpu']                                   */
    uint8_t cpu_numa[NHD_MAX_GROUPS + 1];  /* mapping['cpu'] (last used entry = misc cores)    */
    uint8_t nic_numa[NHD_MAX_GROUPS];      /* mapping['nic'][g][0]                             */
    uint8_t nic_idx[NHD_MAX_GROUPS];       /* mapping['nic'][g][1] (per-NUMA NodeNic.idx)      */
    uint8_t nic_list_index[NHD_MAX_GROUPS];/* index of that NIC in Node.nics                   */
    uint8_t claimed_nics[NHD_MAX_GROUPS];  /* list({x[0] for x in nic_list}), CPython set order */
    uint8_t pad_[3];
    uint8_t gpu_index[NHD_MAX_POD_GPUS];   /* index in Node.gpus per requested GPU, group-major */
    /* logical core ids in canonical order: per group [feeder cores of gpu 0..][proc cores]
     * [helper cores]; then the top-level misc cores (Node.py:728-811). */
    uint8_t cores[NHD_MAX_POD_CORES];
} nhd_binding;

/* Solver parameters: the module constants of nhd/Node.py:18-20,107. */
typedef struct nhd_params {
    double   nic_bw_avail_percent;   /* NIC_BW_AVAIL_PERCENT (0.9)                             */
    double   min_busy_secs;          /* Node.MIN_BUSY_SECS (30.0)                              */
    int32_t  enable_sharing;         /* ENABLE_SHARING; only 0 is supported                    */
    int32_t  n_speed_classes;
    double   speed_gbps[NHD_MAX_SPEED_CLASSES]; /* NodeNic.speed (= label Mb/s / 1e3) per class */
    int32_t  device;                 /* CUDA device ordinal                                    */
    int32_t  rank;                   /* node-shard rank, 0 when single GPU                     */
    int32_t  world_size;             /* number of GPUs sharing the node set                    */
    int32_t  reserved_;              /* 0.  Test hook: low byte 1 = the general one-warp sweep only, 2 = never sweep the two pod
                                      * classes side by side; bit 8 = no standing decisions, bit 9 = same as 2, bit 10 = no direct-path tables;
                                      * all settings produce identical bindings (tests/test_gpu_parity.py)      */
    uint8_t  nccl_unique_id[128];    /* from nhd_nccl_unique_id() on rank 0; unused if world_size==1 */
} nhd_params;

/* per-call device timings of the last nhd_solve_batch (CUDA events, ms) */
typedef struct nhd_timing {
    float filter_ms;             /* snapshot predicate kernel                                  */
    float exchange_ms;           /* NCCL all-gather + slot unpack (0 when world_size == 1)     */
    float sweep_ms;              /* select + assign sweep kernel                               */
    float total_ms;              /* first launch to last kernel end                            */
    int32_t n_types;             /* distinct pod descriptors in the batch                      */
    int32_t n_launches;          /* kernels launched by the call                               */
} nhd_timing;

typedef struct nhd_handle nhd_handle;

void    nhd_default_params(nhd_params* p);
int32_t nhd_nccl_unique_id(uint8_t out[128]);
/* (nodes x distinct pod types of a batch) from which world_size > 1 handles split the snapshot filter over the ranks
 * and exchange the results with one all-gather; smaller batches are filtered whole by every rank with no collective
 * (the reference has no counterpart: it is one process, NHDScheduler.py:43).  NHD_SHARD_MIN_PAIRS in the environment
 * — the same on every rank — overrides the default (2^21) for handles created afterwards. */
int64_t nhd_shard_min_pairs(void);
int32_t nhd_create(const nhd_params* p, nhd_handle** out);
int32_t nhd_destroy(nhd_handle* h);
const char* nhd_last_error(const nhd_handle* h);

/* Page-locked host buffers: records / pods / bindings placed here move to and from the device
 * without a staging copy (anything else is staged internally). */
int32_t nhd_alloc_pinned(uint64_t bytes, void** out);
int32_t nhd_free_pinned(void* p);

/* Host-side validation of wire records against the limits above (nhd_load_nodes runs the same
 * check on the device). */
int32_t nhd_validate_node(const nhd_node_rec* rec);
int32_t nhd_validate_pod(const nhd_pod* pod);

/* Full upload (start-up, ResetResources; NHDScheduler.py:74-105,146-159). */
int32_t nhd_load_nodes(nhd_handle* h, int32_t n_nodes, const nhd_node_rec* recs);
/* Claim / release / cordon / maintenance / group deltas between batches
 * (NHDScheduler.py:107-205,533-570): overwrite records idx[0..n). */
int32_t nhd_update_nodes(nhd_handle* h, int32_t n, const int32_t* idx, const nhd_node_rec* recs);
/* Download the current records [first, first+n). */
int32_t nhd_read_nodes(nhd_handle* h, int32_t first, int32_t n, nhd_node_rec* out);

/* Snapshot / restore of the device mirror (device-to-device; used by benchmarks
 * to replay a batch from the same cluster state).  A restore brings back the snapshot's
 * records with their hardware classes and tuple limits, updates since the snapshot included. */
int32_t nhd_snapshot(nhd_handle* h);
int32_t nhd_restore(nhd_handle* h);

/*
 * Solve a batch with sequential semantics.  now[i] is the value
 * time.monotonic() would return while pod i is scheduled (Node.py:845,848).
 * Host buffers in, host buffers out; the device mirror is updated in place.
 */
int32_t nhd_solve_batch(nhd_handle* h, int32_t n_pods, const nhd_pod* pods,
                        const double* now, nhd_binding* out);

/*
 * The three phases of nhd_solve_batch, separately callable so that a caller (or a
 * benchmark) can keep a batch resident in HBM:
 *   nhd_stage_batch    validate, de-duplicate descriptors into pod types, host -> device
 *   nhd_solve_staged   launch the kernels on the staged batch (asynchronous)
 *   nhd_fetch_bindings wait, device -> host
 * nhd_sync only waits (bindings stay on the device).
 */
int32_t nhd_stage_batch(nhd_handle* h, int32_t n_pods, const nhd_pod* pods, const double* now);
int32_t nhd_solve_staged(nhd_handle* h);
int32_t nhd_fetch_bindings(nhd_handle* h, nhd_binding* out);
int32_t nhd_sync(nhd_handle* h);

/* Debug / tests: run only the snapshot predicate kernel on the staged batch, so that
 * nhd_read_filter returns the bitmaps before the sweep edits them. */
int32_t nhd_run_filter_only(nhd_handle* h);

int32_t nhd_last_timing(const nhd_handle* h, nhd_timing* out);

/*
 * Why the pods of the last solved batch that got NHD_NO_CANDIDATE found no node.  For such a pod i every loaded
 * node n gets a reason NHD_WHY_*: the first stage of the reference that drops n, on the cluster as pod i saw it —
 * the batch-start records plus what pods 0..i-1 of the batch did (cores, GPUs, NICs, hugepages and the busy stamp
 * now[j] of a placement; the busy stamp of a failed assignment), at clock now[i].
 *   nhd_explain_batch  counts[i * NHD_WHY_COUNT + r] = nodes with reason r for pod i; a NO_CANDIDATE row sums to
 *                      n_nodes, every other row is zero.  counts holds n_pods * NHD_WHY_COUNT entries.
 *   nhd_explain_pod    node_reason[n] for one pod (n_nodes bytes); NHD_WHY_NONE everywhere when the pod's status
 *                      is not NHD_NO_CANDIDATE.
 * The batch-start state is read from the handle's snapshot, so both need the sequence
 *     nhd_snapshot -> nhd_stage_batch -> nhd_solve_staged (or nhd_solve_batch)
 * with nothing else changing the mirror in between or since (no load / update / restore / other stage or solve);
 * otherwise they return NHD_ERR_STATE.  Neither changes the mirror, the bindings or the filter bitmaps, and neither
 * enters a collective (every rank holds all records).  They wait for the device before returning.
 */
int32_t nhd_explain_batch(nhd_handle* h, uint32_t* counts);
int32_t nhd_explain_pod(nhd_handle* h, int32_t pod, uint8_t* node_reason);

/*
 * Where each pod would go on its own, without placing anything: the reference's Matcher.FindNode (Matcher.py:27-63),
 * which has no side effects, plus what SetPhysicalIdsFromMapping would take on that node.
 *   NHD_QUERY_MIRROR    the records as they are now
 *   NHD_QUERY_SNAPSHOT  the records of the last nhd_snapshot
 * out[i] is byte for byte the binding nhd_solve_batch(h, 1, &pods[i], &now[i], ...) would return on the chosen
 * records: status, node, mapping, core ids, GPU indices, NIC indices and claim order of pod i ALONE.  Pods do not
 * see each other.  Nothing is written: not the mirror, the snapshot, the staged batch or its bindings, the filter
 * bitmaps or the explanation state; nhd_explain_* and nhd_fetch_bindings of the last batch stay valid across a
 * query.  NHD_QUERY_SNAPSHOT needs a snapshot with no nhd_load_nodes / nhd_update_nodes since it (solves, stages and
 * restores are fine), otherwise NHD_ERR_STATE.  Pods are validated as by nhd_stage_batch (NHD_ERR_INVALID /
 * NHD_ERR_UNSUPPORTED naming the pod index, tuple limits included).  No collective: every rank holds all records and
 * may call alone.  Waits for the device before returning.
 */
#define NHD_QUERY_MIRROR        0
#define NHD_QUERY_SNAPSHOT      1
int32_t nhd_query_batch(nhd_handle* h, int32_t source, int32_t n_pods, const nhd_pod* pods,
                        const double* now, nhd_binding* out);

/*
 * A dry run of a batch: where the pods would go scheduled in order, each seeing the ones before it, with nothing
 * placed.  source is NHD_QUERY_MIRROR or NHD_QUERY_SNAPSHOT, under the same rule as nhd_query_batch.  The nodes
 * excluded[0..n_excluded) are taken as if NHD_NODE_MAINTENANCE were set on their records (Matcher.py:73: what a
 * maintenance start does); an index outside [0, n_nodes) is NHD_ERR_INVALID, a duplicate counts once.
 *   out[i]         byte for byte what nhd_solve_batch(h, n_pods, pods, now, out) would return on the chosen records
 *                  with the excluded nodes so marked;
 *   why_counts     (may be NULL) n_pods * NHD_WHY_COUNT entries: what nhd_explain_batch would return after that solve
 *                  (an excluded node that passes the group and active stages counts as NHD_WHY_MAINTENANCE).
 * Pods are validated and refused as by nhd_stage_batch, naming the pod index; the tuple limits are judged as that solve
 * would judge them, without the excluded nodes.  Nothing is written that a caller can observe: not the mirror, the
 * snapshot, the staged batch, its bindings, filter bitmaps or explanations, nhd_last_timing or nhd_debug_counters.  No
 * collective: every rank holds all records, filters the whole cluster and may call alone (the bindings do not depend
 * on sharding).  Waits for the device before returning.
 */
int32_t nhd_plan_batch(nhd_handle* h, int32_t source, int32_t n_excluded, const int32_t* excluded,
                       int32_t n_pods, const nhd_pod* pods, const double* now,
                       nhd_binding* out, uint32_t* why_counts);

/*
 * Many independent dry runs in one call: "which of these nodes (or racks) could be taken down, each on its own?".
 * Scenario s excludes excluded[excl_start[s] .. excl_start[s+1]) and plans pods[pod_start[s] .. pod_start[s+1]) with
 * now[] of the same rows; both offset arrays hold n_scenarios + 1 entries, start at 0 and never go down.
 *   out[pod_start[s] .. pod_start[s+1])  when scenario_status[s] == NHD_OK: byte for byte what
 *                  nhd_plan_batch(h, source, n_excl_s, excl_s, n_pods_s, pods_s, now_s, out_s, NULL) would return.
 *                  Scenarios do not see each other; the pods inside one see the earlier ones, in order.
 *   scenario_status[s], scenario_pod[s]  NHD_OK and -1, or the refusal nhd_plan_batch would give that scenario
 *                  (NHD_ERR_INVALID / NHD_ERR_UNSUPPORTED: a descriptor nhd_validate_pod rejects, a non-finite clock,
 *                  the tuple limits) and the index inside the scenario of the pod it names.  The out rows of a refused
 *                  scenario are not written.
 * source is NHD_QUERY_MIRROR or NHD_QUERY_SNAPSHOT, under the same rule as nhd_query_batch.  Unlike nhd_plan_batch the
 * tuple limits are judged against every schedulable node of the cluster, the excluded ones included: one filter on the
 * unchanged records serves every scenario, and it enumerates the NUMA tuples of the excluded nodes too.  Exclusions can
 * only lower the largest NUMA count, so this refuses only scenarios that nhd_plan_batch accepts because of their
 * exclusions; plan such a scenario with nhd_plan_batch.
 * Malformed arguments make the whole call NHD_ERR_INVALID: a null pointer, offsets that do not start at 0 or go down,
 * an excluded index outside [0, n_nodes); a duplicate exclusion counts once.  Nothing is written that a caller can
 * observe (the same list as nhd_plan_batch), no collective is entered (any rank may call alone), and the call waits
 * for the device before returning.  Explanations are not part of it: nhd_plan_scenarios_explained gives them.
 * Meant for many small scenarios (the pods of one node or one rack): one warp runs each, and a pod's cost grows with
 * the number of nodes its scenario's earlier pods reached.  A large single batch belongs to nhd_plan_batch.
 */
int32_t nhd_plan_scenarios(nhd_handle* h, int32_t source, int32_t n_scenarios,
                           const int32_t* excl_start, const int32_t* excluded,
                           const int32_t* pod_start, const nhd_pod* pods, const double* now,
                           nhd_binding* out, int32_t* scenario_status, int32_t* scenario_pod);

/*
 * nhd_plan_scenarios with replaced records and exclusions that end: "if these nodes were drained and put back in
 * service, would their pods place elsewhere, and would the pending pods then place?".  Scenario s, with its pods
 * numbered k = 0 .. n_s - 1 inside it:
 *   - for every e in [edit_start[s], edit_start[s+1]), node edit_node[e] has record edit_rec[e] for the whole scenario;
 *   - its excluded nodes are in maintenance for its pods k < lift_at[s] and back in service from pod lift_at[s] on,
 *     each with the flags of its record (the replacement if it has one) plus what the scenario's earlier pods did to it.
 *   out[pod_start[s] .. pod_start[s+1])  when scenario_status[s] == NHD_OK: byte for byte what nhd_solve_batch would
 *                  return on a scratch copy of the source records with (1) the edits applied, (2) NHD_NODE_MAINTENANCE
 *                  set on the excluded nodes, (3) pods [0, lift_at[s]) solved, (4) the excluded nodes' flags put back,
 *                  (5) pods [lift_at[s], n_s) solved.
 * lift_at == NULL, or lift_at[s] == n_s, keeps the exclusions to the end; edit_start == NULL means no edits (then
 * edit_node and edit_rec are not read).  With neither, the call is nhd_plan_scenarios.  Refusals are per scenario as
 * there, with the tuple limits judged against the larger of the cluster's largest schedulable NUMA count and the
 * n_numa of every edit record of the call.  Besides nhd_plan_scenarios' malformed arguments, the whole call is
 * NHD_ERR_INVALID for edit offsets that do not start at 0 or go down, an edit_node outside [0, n_nodes), a node
 * edited twice in one scenario, an edit record nhd_validate_node rejects, and a lift_at[s] outside [0, n_s].  Side effects, collectives and waiting as for nhd_plan_scenarios.
 */
int32_t nhd_plan_scenarios_edited(nhd_handle* h, int32_t source, int32_t n_scenarios,
                                  const int32_t* excl_start, const int32_t* excluded, const int32_t* lift_at,
                                  const int32_t* edit_start, const int32_t* edit_node, const nhd_node_rec* edit_rec,
                                  const int32_t* pod_start, const nhd_pod* pods, const double* now,
                                  nhd_binding* out, int32_t* scenario_status, int32_t* scenario_pod);

/*
 * nhd_plan_scenarios_edited with reasons: "why does this planned pod find no node?".  Arguments, validation, refusals,
 * tuple limits, bindings, side effects (none observable), collectives and waiting are exactly those of
 * nhd_plan_scenarios_edited; with why_counts == NULL the call is nhd_plan_scenarios_edited.
 *   why_counts     pod_start[n_scenarios] * NHD_WHY_COUNT entries.  For an accepted scenario s and its pod k with status
 *                  NHD_NO_CANDIDATE, row pod_start[s] + k counts per reason the nodes whose first dropping stage is that
 *                  reason, on the scenario's records as that pod saw them: the source records with s's edits, with its
 *                  earlier pods' effects (placements, and the busy stamp of a failed assignment) and with its excluded
 *                  nodes in maintenance while k < lift_at[s], at clock now[pod_start[s] + k].  That is the row
 *                  nhd_explain_batch would give the pod after the five steps of nhd_plan_scenarios_edited, taken on the
 *                  records at the start of the pod's own phase.  Rows of the other pods of accepted scenarios are zero;
 *                  rows of refused scenarios are not written.
 * A NO_CANDIDATE row that would not sum to n_nodes, or a node passing every stage for such a pod, is NHD_ERR_STATE.
 */
int32_t nhd_plan_scenarios_explained(nhd_handle* h, int32_t source, int32_t n_scenarios,
                                     const int32_t* excl_start, const int32_t* excluded, const int32_t* lift_at,
                                     const int32_t* edit_start, const int32_t* edit_node, const nhd_node_rec* edit_rec,
                                     const int32_t* pod_start, const nhd_pod* pods, const double* now,
                                     nhd_binding* out, int32_t* scenario_status, int32_t* scenario_pod,
                                     uint32_t* why_counts);

/*
 * nhd_plan_scenarios_explained on a grown cluster: "would these added nodes let the pending pods place?".  Scenario s
 * also adds the records add_rec[a], a in [add_start[s], add_start[s+1]):
 *   - added node a joins the node order right before source node add_at[a] (add_at[a] == n_nodes: after the last
 *     node); added nodes with the same add_at keep their array order; add_at never goes down inside a scenario;
 *   - an added node is in service for the whole scenario: exclusions, edits and lift_at refer to source nodes only.
 *   out[pod_start[s] .. pod_start[s+1])  when scenario_status[s] == NHD_OK: byte for byte what nhd_solve_batch would
 *                  return after the five steps of nhd_plan_scenarios_edited taken on a scratch copy of the source
 *                  records with the edits applied and the added records inserted at their positions, every node index
 *                  mapped back: a source node to its index, added node a to n_nodes + a (a the call-wide index into
 *                  add_rec, also when refused scenarios are left out).
 *   why_counts     (may be NULL) as for nhd_plan_scenarios_explained, counted over the scenario's grown node list: a
 *                  NO_CANDIDATE row sums to n_nodes + add_start[s+1] - add_start[s].
 * The tuple limits are judged against the largest of the cluster's largest schedulable NUMA count, the n_numa of every
 * edit record and the n_numa of every added record of the call.  Besides nhd_plan_scenarios_explained's malformed
 * arguments, the whole call is NHD_ERR_INVALID for add offsets that do not start at 0 or go down, an add_at outside
 * [0, n_nodes] or going down inside a scenario, an added record nhd_validate_node rejects, and an added record with a
 * NIC of a speed class at or above the handle's n_speed_classes (the handle holds no capacity for it).  add_start ==
 * NULL means no additions (add_at and add_rec are not read): the call is nhd_plan_scenarios_explained.  Side effects
 * (none observable), collectives and waiting as for nhd_plan_scenarios.
 */
int32_t nhd_plan_scenarios_grown(nhd_handle* h, int32_t source, int32_t n_scenarios,
                                 const int32_t* excl_start, const int32_t* excluded, const int32_t* lift_at,
                                 const int32_t* edit_start, const int32_t* edit_node, const nhd_node_rec* edit_rec,
                                 const int32_t* add_start, const int32_t* add_at, const nhd_node_rec* add_rec,
                                 const int32_t* pod_start, const nhd_pod* pods, const double* now,
                                 nhd_binding* out, int32_t* scenario_status, int32_t* scenario_pod,
                                 uint32_t* why_counts);

/*
 * nhd_plan_scenarios_grown over several pending scans: "which pods get in at a later scan, and which never do?".  The
 * scheduler retries every pod still pending at each scan, and a GPU node that took a pod (or failed an assignment) less
 * than min_busy_secs earlier takes no GPU pod, so one scan cannot tell "never fits" from "fits at the next scan".
 * Scenario s has R_s = round_start[s+1] - round_start[s] later rounds; round r >= 1 runs at clock
 * round_clock[round_start[s] + r - 1].  After the five steps of nhd_plan_scenarios_grown (round 0), for r = 1 .. R_s
 * the pods of s whose latest binding is not NHD_PLACED are solved in scenario order as one nhd_solve_batch at that
 * round's clock, on the records the previous round left; a round with no such pod does nothing.
 *   - exclusions still held for the last pod of round 0 (lift_at NULL or lift_at[s] == n_s) stay held in every later
 *     round; exclusions lifted during round 0 stay lifted; edits and added nodes hold for the whole scenario;
 *   out            byte for byte each pod's last attempt, node indices mapped back as for nhd_plan_scenarios_grown;
 *   pod_round      (may be NULL) pod_start[n_scenarios] entries: the round that placed the pod, or R_s if none did;
 *   why_counts     (may be NULL) for a pod whose last attempt is NHD_NO_CANDIDATE, the row nhd_explain_batch would give
 *                  at the start of that attempt, at that round's clock, over the scenario's grown node list; other rows
 *                  zero.
 * Besides nhd_plan_scenarios_grown's malformed arguments, the whole call is NHD_ERR_INVALID for round offsets that do
 * not start at 0 or go down, a non-finite round clock, round clocks that go down inside a scenario, and a round clock
 * earlier than a now[] of its scenario (a monotonic clock never goes back).  The busy test is now - busy_time <
 * min_busy_secs in fp64: give the clocks exactly as the caller's clock would read them, each the previous one plus the
 * period, not t0 + r * period.  round_start == NULL means no rounds (round_clock is not read): the call is
 * nhd_plan_scenarios_grown and pod_round, if given, is all zero.  Refusals per scenario, tuple limits, side effects
 * (none observable), collectives and waiting as for nhd_plan_scenarios_grown.  Each scenario's pods may touch up to
 * min(n_s * (1 + R_s), n_nodes) nodes besides its edited and added ones: device scratch grows with that bound.
 */
int32_t nhd_plan_scenarios_rounds(nhd_handle* h, int32_t source, int32_t n_scenarios,
                                  const int32_t* excl_start, const int32_t* excluded, const int32_t* lift_at,
                                  const int32_t* edit_start, const int32_t* edit_node, const nhd_node_rec* edit_rec,
                                  const int32_t* add_start, const int32_t* add_at, const nhd_node_rec* add_rec,
                                  const int32_t* pod_start, const nhd_pod* pods, const double* now,
                                  const int32_t* round_start, const double* round_clock,
                                  nhd_binding* out, int32_t* scenario_status, int32_t* scenario_pod,
                                  uint32_t* why_counts, int32_t* pod_round);

/*
 * nhd_plan_batch over several pending scans: "the queue I have now, on the cluster I have now: which pods get in at a
 * later scan, and which never do?".  One large batch, solved by the batch path at every scan (nhd_plan_scenarios_rounds
 * runs each scenario on one warp and is meant for many small ones).  Round 0 is nhd_plan_batch(h, source, n_excluded,
 * excluded, n_pods, pods, now, ...).  For r = 1 .. n_rounds the pods whose latest binding is not NHD_PLACED are solved
 * in their original order as one nhd_solve_batch at clock round_clock[r-1], on the records the previous round left
 * (placements, and the busy stamp of a failed assignment, committed to the plan's own copy); a round with no such pod
 * does nothing.  The excluded nodes stay in maintenance in every round.
 *   out[i]         byte for byte pod i's last attempt;
 *   pod_round      (may be NULL) n_pods entries: the round that placed the pod, or n_rounds if none did;
 *   why_counts     (may be NULL) n_pods * NHD_WHY_COUNT entries: for a pod whose last attempt is NHD_NO_CANDIDATE, the
 *                  row nhd_explain_batch would give for that attempt (the records at the start of that round plus that
 *                  round's earlier pods, at the round's clock); all other rows zero.
 * Bindings, pod_round and why_counts equal those of nhd_plan_scenarios_rounds called with this one scenario, its
 * exclusions held to the end (lift_at NULL), no edits and no additions; the one difference is nhd_plan_batch's: the
 * tuple limits are judged without the excluded nodes.  n_rounds == 0 is nhd_plan_batch (round_clock is not read,
 * pod_round, if given, is all zero).
 * Refused as nhd_plan_batch refuses, and NHD_ERR_INVALID for n_rounds < 0, a NULL round_clock with n_rounds > 0, a
 * non-finite round clock, round clocks that go down, and a first round clock earlier than a now[] (a monotonic clock
 * never goes back).  The busy test is now - busy_time < min_busy_secs in fp64: give the clocks exactly as the caller's
 * clock would read them, each the previous one plus the period, not t0 + r * period.  A node passing every stage for a
 * NO_CANDIDATE pod is NHD_ERR_STATE.  Nothing is written that a caller can observe (the list of nhd_plan_batch), no
 * collective is entered (any rank may call alone), and the call waits for the device before returning.
 */
int32_t nhd_plan_batch_rounds(nhd_handle* h, int32_t source, int32_t n_excluded, const int32_t* excluded,
                              int32_t n_pods, const nhd_pod* pods, const double* now,
                              int32_t n_rounds, const double* round_clock,
                              nhd_binding* out, uint32_t* why_counts, int32_t* pod_round);

/* One deployed pod given back between two scans of a forecast (ReleasePodResources, NHDScheduler.py:174-205), 88 bytes. */
typedef struct nhd_release {
    int32_t  node;                        /* node index in load order                                         */
    int32_t  round;                       /* 1 .. n_rounds: lands after round - 1 and before round             */
    double   clock;                       /* time.monotonic() at the release; Node.SetBusy stamps it (:205)   */
    uint64_t cores[4];                    /* bit c: Node.cores[c].used = False (Node.py:590-619)              */
    uint16_t gpus;                        /* bit i: Node.gpus[i].used = False                                 */
    uint8_t  pad_[2];
    int32_t  hugepages_gb;                /* added to free_hugepages_gb when > 0 (Node.py:634-635)            */
    uint8_t  nic_pairings[NHD_MAX_NICS];  /* per Node.nics[i]: nic_core_pairing entries, each pods_used -= 1  */
} nhd_release;

/*
 * nhd_plan_batch_rounds with running pods finishing between the scans: "these deployed pods end at about these times:
 * when does each pending pod get in, and on which node?".  Rounds, pods, exclusions and clocks are those of
 * nhd_plan_batch_rounds.  Before round r >= 1 the releases with round == r are applied, in array order, to the plan's
 * own copy of the records: their core and GPU bits cleared, hugepages_gb added when > 0, the NIC counters lowered by
 * nic_pairings, and busy_time = clock (a freed GPU node takes no GPU pod for min_busy_secs after the release).
 * The records carry one in-use bit per NIC; the reference carries a signed counter, NodeNic.pods_used, which a release
 * lowers once per RX/TX pairing (Node.py:621-631) and a claim raises once per distinct NIC (Node.py:644-646), so after a
 * pod with two pairings on one NIC ends the counter sits at -1 and the next claim leaves the NIC free (Node.py:292).
 * The call carries those counters for the nodes tracked[0..n_tracked): pods_used[t * NHD_MAX_NICS + i] is the counter
 * of NIC i of node tracked[t] at plan start.  Every release's node must be tracked; a caller also tracks every node
 * with a negative counter.  On a tracked node a NIC's in-use bit is count > 0 after every release, and every placement
 * raises the count of each NIC in its claimed_nics by 1.
 *   out, pod_round, why_counts   as for nhd_plan_batch_rounds: byte for byte what the reference's scheduler gives,
 *                  every round solved one pod at a time on the records and counters, the releases played between rounds.
 * The batch path differs from that only where a placement claims a tracked NIC whose count is <= -1 before the claim
 * (the solve's commit sets a bit the reference leaves clear).  The call then cuts the round right after that pod: it
 * restores the records the round's segment started from, solves that prefix again with its commit (the solve is
 * deterministic), clears the bit from the count and solves the rest of the round as a new segment at the same clock.
 * Each cut uses up one unit of negative count, so a call makes at most sum(|negative pods_used|) + sum(nic_pairings)
 * cuts, each one more solve of its prefix and one host read.  Only the last round's last attempts are explained, each
 * on the records its segment started from.
 * With n_releases == 0 and n_tracked == 0 the call is nhd_plan_batch_rounds (tracked, pods_used and releases are not
 * read).  Refused as nhd_plan_batch_rounds refuses, and, before anything is placed on the plan's copy, NHD_ERR_INVALID
 * for: n_tracked or n_releases < 0 or their arrays NULL; a tracked node outside [0, n_nodes) or tracked twice; a
 * release round outside [1, n_rounds]; release clocks that go down in array order, are not finite, lie before the
 * clock of the round before theirs (before every now[] for round 1) or after their own round's clock; a release on an
 * untracked node; and, checked on the device against the source records (one word read back), a tracked count whose
 * sign disagrees with the NIC's in-use bit (> 0 exactly when set), a NIC at or beyond n_nics with a non-zero count, a
 * core bit at or beyond the node's logical core count, a GPU bit at or beyond n_gpus, or a pairing on a NIC at or
 * beyond n_nics.  Nothing is written that a caller can observe (the list of nhd_plan_batch), no collective is entered,
 * and the call waits for the device before returning.
 */
int32_t nhd_plan_batch_releases(nhd_handle* h, int32_t source, int32_t n_excluded, const int32_t* excluded,
                                int32_t n_pods, const nhd_pod* pods, const double* now,
                                int32_t n_rounds, const double* round_clock,
                                int32_t n_tracked, const int32_t* tracked, const int16_t* pods_used,
                                int32_t n_releases, const nhd_release* releases,
                                nhd_binding* out, uint32_t* why_counts, int32_t* pod_round);

/*
 * nhd_plan_batch_releases with pods created between the scans, on the batch path: "we submit these 4 000 jobs at 10:05
 * and jobs A and B end at 10:10: when does each one start, and on which node?", one timeline of many pods.  Every
 * argument of nhd_plan_batch_releases keeps its meaning; pod i also has
 *   arrive_round[i]  0: pending at plan start; r in [1, n_rounds]: created in the gap before round r, at clock now[i].
 *                    The round-0 pods come first, and (arrive_round, now) never goes down in pod order.
 * Round 0 solves the round-0 pods as nhd_plan_batch_releases does.  Each gap r >= 1 then plays, merged by clock, the
 * releases of round r and the first attempt of each pod arriving in it, at its now[] (the reference attempts a new pod
 * on its create event); a release goes before an arrival at the same clock, and arrivals keep pod order.  Round r's
 * scan then retries, in pod order at round_clock[r-1], every arrived pod not placed yet, the gap's failed arrivals after
 * the older pods.  A gap's releases are played while a pod is unplaced or has not arrived yet.  The excluded nodes stay
 * in maintenance throughout.
 *   out            the binding of each pod's placing attempt, or else of its last one;
 *   pod_round      (may be NULL) the round r whose arrival or scan placed the pod, or n_rounds if none did;
 *   pod_clock      (may be NULL) the clock of the attempt whose binding is in out: now[i] or a round's clock;
 *   why_counts     (may be NULL) the row at the start of the pod's last attempt, always a scan, as for
 *                  nhd_plan_batch_releases.
 * Identities: with arrive_round NULL the call is nhd_plan_batch_releases byte for byte on out, pod_round and
 * why_counts, pod_clock then now[i] or the clock of the round that made the pod's last attempt.  The call gives the
 * out, pod_round, pod_clock and why_counts of nhd_plan_scenarios_arrivals called with this one timeline as one scenario,
 * its exclusions held throughout (lift_at = n_pods), no edits and no additions; the one difference is the tuple-limit
 * judgement, as between nhd_plan_scenarios and nhd_plan_batch.
 * Each run of a gap's arrivals between two of its releases is solved as one batch at per-pod clocks, with its commit,
 * and cut where a claim meets a negative NIC count exactly as a round is; arrivals add no negative count, so the bound
 * on cuts of nhd_plan_batch_releases holds.
 * Refused as nhd_plan_batch_releases refuses, and, before anything is placed, NHD_ERR_INVALID for an arrive_round
 * outside [0, n_rounds] or going down in pod order, an arrival with n_rounds == 0, arrival clocks going down among the
 * arrivals of one gap, and an arrival clock before the clock of the round before its gap (for gap 1: before a now[] of a
 * round-0 pod) or after its own round's clock.  The rule that no round clock is earlier than a now[] reads the round-0
 * pods only, as does the lower bound of a round-1 release's clock.  Tuple limits are judged as by nhd_plan_batch.
 * Nothing is written that a caller can observe (the list of nhd_plan_batch), no collective is entered, and the call
 * waits for the device before returning.
 */
int32_t nhd_plan_batch_arrivals(nhd_handle* h, int32_t source, int32_t n_excluded, const int32_t* excluded,
                                int32_t n_pods, const nhd_pod* pods, const double* now,
                                int32_t n_rounds, const double* round_clock,
                                int32_t n_tracked, const int32_t* tracked, const int16_t* pods_used,
                                int32_t n_releases, const nhd_release* releases, const int32_t* arrive_round,
                                nhd_binding* out, uint32_t* why_counts, int32_t* pod_round, double* pod_clock);

/*
 * nhd_plan_scenarios_rounds with running pods finishing between the scans, per scenario: "jobs A and B end in about 20
 * minutes: does the queue clear then, or do I also need one more node like this one?", and several departure schedules
 * side by side.  Every argument of nhd_plan_scenarios_rounds keeps its meaning; scenario s also has
 *   - tracked nodes tracked[track_start[s] .. track_start[s+1]) with their signed NIC pod counters at plan start,
 *     pods_used[t * NHD_MAX_NICS + i] for NIC i of tracked[t] (t call-wide), as for nhd_plan_batch_releases;
 *   - releases releases[rel_start[s] .. rel_start[s+1]), round 1 .. R_s.
 * Before round r >= 1, if a pod of s is still unplaced, s's releases with round == r are applied in array order to s's
 * own records and counters: core and GPU bits cleared, hugepages_gb added when > 0, the counters lowered by
 * nic_pairings, busy_time = clock.  On a tracked node a NIC's in-use bit is count > 0 after every release and after
 * every placement, and each placement raises the count of every NIC in its claimed_nics by 1 when that pod commits.
 * Scenarios commit one pod at a time, so unlike nhd_plan_batch_releases nothing is cut or solved again.
 *   out, pod_round  as for nhd_plan_scenarios_rounds, on those records;
 *   why_counts     (may be NULL) as for nhd_plan_scenarios_rounds: the row nhd_explain_batch would give at the start of
 *                  the pod's last attempt.
 * Identities: with track_start and rel_start both NULL (tracked, pods_used and releases are not read) the call is
 * nhd_plan_scenarios_rounds.  One scenario with no edits, no additions and lift_at NULL gives the out and pod_round of
 * nhd_plan_batch_releases with the same pods, round clocks, exclusions, tracked counters and releases, byte for byte;
 * the only difference is the tuple-limit judgement, as between nhd_plan_scenarios and nhd_plan_batch.
 * Releases on a node the scenario edits are out of scope: such a release refuses the call (an edited record replaces
 * the node's whole state, so a caller releasing on it edits the record instead).
 * Besides nhd_plan_scenarios_rounds' malformed arguments, the whole call is NHD_ERR_INVALID, before anything runs, for
 * track or release offsets that do not start at 0 or go down; tracked or pods_used NULL with tracked nodes, releases
 * NULL with releases; a tracked node outside [0, n_nodes) or tracked twice in one scenario; releases in a scenario
 * without rounds, or a release round outside [1, R_s]; release clocks that go down inside a scenario, are not finite,
 * lie before the clock of the round before theirs (for round 1: before a now[] of the scenario) or after their own
 * round's clock; a release on a node its scenario does not track, or edits; and, checked on the device against the
 * source records (one word read back), a tracked count whose sign disagrees with the NIC's in-use bit (> 0 exactly
 * when set), a non-zero count on a NIC at or beyond n_nics, or a release's core, GPU or pairing bit beyond its node's
 * logical cores, n_gpus or n_nics.  Tuple limits, refusals per scenario, side effects (none observable), collectives
 * (none) and waiting as for nhd_plan_scenarios_rounds.  Each scenario's slot bound grows by its distinct released
 * nodes, and the device holds its tracked nodes' counts: n_tracked_s * NHD_MAX_NICS int32.
 */
int32_t nhd_plan_scenarios_releases(nhd_handle* h, int32_t source, int32_t n_scenarios,
                                    const int32_t* excl_start, const int32_t* excluded, const int32_t* lift_at,
                                    const int32_t* edit_start, const int32_t* edit_node, const nhd_node_rec* edit_rec,
                                    const int32_t* add_start, const int32_t* add_at, const nhd_node_rec* add_rec,
                                    const int32_t* pod_start, const nhd_pod* pods, const double* now,
                                    const int32_t* round_start, const double* round_clock,
                                    const int32_t* track_start, const int32_t* tracked, const int16_t* pods_used,
                                    const int32_t* rel_start, const nhd_release* releases,
                                    nhd_binding* out, int32_t* scenario_status, int32_t* scenario_pod,
                                    uint32_t* why_counts, int32_t* pod_round);

/*
 * nhd_plan_scenarios_releases with pods created between the scans, per scenario: "we submit these 200 jobs at 10:05 and
 * jobs A and B end at 10:10: when does each one start, and on which node?".  Every argument of
 * nhd_plan_scenarios_releases keeps its meaning; pod i also has
 *   arrive_round[i]  0: pending at plan start; r in [1, R_s]: created in the gap before round r, at clock now[i].  The
 *                    round-0 pods come first in the scenario's pod order, and (arrive_round, now) never goes down in
 *                    pod order.
 * Per scenario: round 0 solves the round-0 pods in order, each at its now[].  Each gap r >= 1 then plays, merged by
 * clock, the scenario's releases of round r and the first attempt of each pod arriving in it, solved alone at its
 * now[] (the reference attempts a new pod on its create event); a release goes before an arrival at the same clock,
 * and arrivals keep pod order.  Round r's scan then retries, in pod order at the round's clock, every arrived pod
 * (arrive_round <= r) not placed yet, the gap's failed arrivals included.  A gap's releases are played while a pod of
 * the scenario is unplaced or has not arrived yet.
 *   out            the binding of each pod's placing attempt, or else of its last one;
 *   pod_round      the round r whose arrival or scan placed the pod, or R_s if none did;
 *   pod_clock      (may be NULL) the clock of the attempt whose binding is in out: now[i] or a round's clock;
 *   why_counts     (may be NULL) as for nhd_plan_scenarios_releases: the row at the start of the pod's last attempt,
 *                  always a scan (every gap is followed by its scan).
 * Exclusions: lift_at[s] must be <= n0_s, the number of round-0 pods (the maintenance ends after round 0 from that
 * pod on), or == n_s (held throughout).
 * Identities: with arrive_round NULL the call is nhd_plan_scenarios_releases byte for byte, pod_clock then now[i] or
 * the clock of the round that made the pod's last attempt.  A scenario whose pods all arrive in gap 1 and which has
 * no release of round 1 gives the out, why_counts and pod_clock of nhd_plan_scenarios_releases on the same pods as
 * round-0 pods at the same now[], and its pod_round with 0 read as 1.
 * Besides nhd_plan_scenarios_releases' malformed arguments, the whole call is NHD_ERR_INVALID, before anything runs,
 * for an arrive_round outside [0, R_s] or going down in pod order, an arrival in a scenario without rounds, arrival
 * clocks going down among the arrivals of one gap, an arrival clock before the clock of the round before its gap (for
 * gap 1: before a now[] of a round-0 pod) or after its own round's clock, and a lift_at other than the two above.
 * The rule that no round clock is earlier than a now[] of its scenario reads the round-0 pods only, as does the lower
 * bound of a round-1 release's clock.  Each pod is attempted at most 1 + R_s times, so the slot bound of
 * nhd_plan_scenarios_releases holds.  Tuple limits, refusals per scenario, side effects (none observable), collectives
 * (none) and waiting as for nhd_plan_scenarios_releases.
 */
int32_t nhd_plan_scenarios_arrivals(nhd_handle* h, int32_t source, int32_t n_scenarios,
                                    const int32_t* excl_start, const int32_t* excluded, const int32_t* lift_at,
                                    const int32_t* edit_start, const int32_t* edit_node, const nhd_node_rec* edit_rec,
                                    const int32_t* add_start, const int32_t* add_at, const nhd_node_rec* add_rec,
                                    const int32_t* pod_start, const nhd_pod* pods, const double* now,
                                    const int32_t* round_start, const double* round_clock,
                                    const int32_t* track_start, const int32_t* tracked, const int16_t* pods_used,
                                    const int32_t* rel_start, const nhd_release* releases, const int32_t* arrive_round,
                                    nhd_binding* out, int32_t* scenario_status, int32_t* scenario_pod,
                                    uint32_t* why_counts, int32_t* pod_round, double* pod_clock);

/* Per-pod-type feasibility bitmaps of the last solve's snapshot filter
 * (debug / tests): words[t * words_per_type + w], bit b of word w = node 64*w+b. */
int32_t nhd_read_filter(nhd_handle* h, int32_t* n_types, int32_t* words_per_type,
                        uint64_t* words, int64_t capacity_words, int32_t* pod_type, int32_t n_pods);

/* Debug: 64 words of per-phase cycle accumulators / counters of the last sweep; only non-zero
 * in libraries built with -DNHD_PROFILE. */
int32_t nhd_debug_counters(nhd_handle* h, uint64_t* out64);

/* ---- node ingest (host side, no GPU): NFD label dictionary -> nhd_node_rec --------------------
 * Replaces Node.ParseLabels (nhd/Node.py:468-487: InitGroups :312, InitMaintenance :324, InitCores :328,
 * InitNics :378, InitGpus :428, InitMisc :440) + Node.SetHugepages (:489-493) for a node the scheduler has
 * just discovered (nhd/NHDScheduler.py:122-140), and the packing of the resulting Node object.
 * An nhd_ingest holds the two cluster-wide dictionaries the records refer to: node-group names -> bits of
 * group_mask, NIC link speeds -> speed classes (= nhd_params.speed_gbps).  What the placement loop does not
 * need (interface names, MACs, the gateway string) stays with the caller, addressed by label position. */
typedef struct nhd_ingest nhd_ingest;

typedef struct nhd_node_aux {
    int32_t data_vlan;                     /* DATA_PLANE_VLAN                (Node.py:441-446)   */
    int32_t res_hugepages_gb;              /* RES_HUGEPAGES_GB, 0 if absent  (Node.py:451-453)   */
    int32_t n_reserved_cores;              /* len(Node.reserved_cores)       (Node.py:368-371)   */
    int32_t gw_label;                      /* index of the DATA_DEFAULT_GW label                  */
    int32_t gpu_device_id[NHD_MAX_GPUS];   /* Node.gpus[i].device_id, -1 beyond n_gpus            */
    int32_t nic_label[NHD_MAX_NICS];       /* index of the label Node.nics[i] came from, -1 beyond n_nics */
} nhd_node_aux;

int32_t nhd_ingest_create(nhd_ingest** out);
int32_t nhd_ingest_destroy(nhd_ingest* g);
/* keys / values: the node's labels in dictionary order (NIC / GPU list order follows label order).
 * NHD_ERR_LABELS: the reference's ParseLabels returns False; NHD_ERR_INVALID: it would raise;
 * NHD_ERR_UNSUPPORTED: beyond NHD_MAX_*.  aux may be NULL. */
int32_t nhd_ingest_node(nhd_ingest* g, int32_t n_labels, const char* const* keys, const char* const* values,
                        int32_t active, int32_t hugepages_alloc_gb, int32_t hugepages_free_gb,
                        nhd_node_rec* rec, nhd_node_aux* aux);
/* '.'-joined group names (the NHD_GROUP label / pod group annotation) -> group_mask bits */
int32_t nhd_ingest_group_mask(nhd_ingest* g, const char* dotted_names, int32_t create, uint64_t* mask);
/* speed classes seen so far, for nhd_params.speed_gbps */
int32_t nhd_ingest_speed_table(const nhd_ingest* g, double out[NHD_MAX_SPEED_CLASSES], int32_t* n_classes);

/* ---- node statistics from packed records (host side) ------------------------------------------
 * What NHDScheduler.GetBasicNodeStats (nhd/NHDScheduler.py:355-378) reads off a Node, for records that came
 * back from the device mirror (nhd_read_nodes): the counters the packed state carries.  totalhuge_gb,
 * totalpods and the per-NIC used speeds are not part of the placement state and stay with the caller. */
typedef struct nhd_node_stats {
    int32_t freegpu;                       /* Node.GetFreeGpuCount()      (Node.py:235-237) */
    int32_t totalgpu;                      /* Node.GetTotalGPUs()         (Node.py:239-241) */
    int32_t freecpu;                       /* Node.GetFreeCpuCoreCount(): logical cores, with SMT only those whose
                                            * sibling is free too         (Node.py:225-233) */
    int32_t totalcpu;                      /* Node.GetTotalCPUs() = len(Node.cores)         (Node.py:243-245) */
    int32_t freehuge_gb;                   /* Node.GetFreeHugepages()     (Node.py:171-173) */
    int32_t active;                        /* Node.GetNodeActive()        (Node.py:163-165) */
    int32_t maintenance;
    int32_t nics_in_use;                   /* NICs with pods_used > 0 */
    int32_t free_cores_numa[NHD_MAX_NUMA]; /* Node.GetFreeCpuCores(): free physical cores per NUMA node (Node.py:250-264) */
    int32_t free_gpus_numa[NHD_MAX_NUMA];  /* Node.GetFreeNumaGPUs()      (Node.py:456-462) */
} nhd_node_stats;
int32_t nhd_node_stats_from_records(int32_t n, const nhd_node_rec* recs, nhd_node_stats* out);

#ifdef __cplusplus
}
#endif
#endif /* NHD_B200_H */
