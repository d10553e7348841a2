/*
 * explain_oracle.c — ORACLE for nhd_explain_batch / nhd_explain_pod (test infrastructure only).
 *
 * For one pod and a cluster state, the first stage of the reference that drops each node, found by running the
 * oracle's own statement-by-statement restatement of those stages (oracle/nhd_oracle.c, included below so that its
 * file-local stage functions are reachable without changing it) one after another and stopping at the first that
 * drops the node:
 *   NHDScheduler.InitialNodeFilter   nhd/NHDScheduler.py:240 (groups), :241 (active)
 *   Matcher.FilterPodResources       nhd/Matcher.py:73 (maintenance), :78 (hugepages)
 *   Matcher.FilterNumaTopology       :107-111 (busy window), :132 (GPUs), :214 (CPU cores), :270 (NICs)
 *   Matcher.IntersectResources       :295-359 (PCI pruning, NUMA intersection)
 * Nothing here is shared with the product (nhd_b200/): candidate lists are materialised and Python set semantics
 * come from pyset_model.c, exactly as for nhd_oracle_solve.
 */
#include "../oracle/nhd_oracle.c"

static int explain_one(const o_node* v, const o_pod* top, double now)
{
    if ((v->groups & top->groups) == 0) return NHD_WHY_GROUP;           /* NHDScheduler.py:240 */
    if (!v->active) return NHD_WHY_INACTIVE;                             /* :241 */
    if (v->maintenance) return NHD_WHY_MAINTENANCE;                      /* Matcher.py:73 */
    if (top->hugepages_gb > v->free_hugepages_gb) return NHD_WHY_HUGEPAGES;   /* :78 */
    int sum = 0;                                                         /* :107-111, ahead of the GPU tuples */
    for (int g = 0; g < top->n_groups; g++) sum += top->g[g].n_gpus;
    if (sum > 0 && node_is_busy(v, now)) return NHD_WHY_BUSY;
    o_filts f;
    memset(&f, 0, sizeof(f));
    int why = NHD_WHY_COUNT;
    if (!filter_gpu_stage(v, top, now, &f)) why = NHD_WHY_GPU;          /* :132 */
    else if (!filter_cpu_stage(v, top, &f)) why = NHD_WHY_CPU;          /* :214 */
    else if (!filter_nic_stage(v, top, &f)) why = NHD_WHY_NIC;          /* :270 */
    else if (!intersect_node(v, top, &f)) why = NHD_WHY_INTERSECT;      /* :353 */
    filts_free(&f);
    return why;
}

/* reason[n] for every node of recs (the state the pod sees) at clock now; NHD_WHY_COUNT = the node passes every stage */
int nhd_oracle_explain(const nhd_oracle_params* params, const double* speed_gbps, int n_nodes, const nhd_node_rec* recs,
                       const nhd_pod* pod, double now, uint8_t* reason)
{
    P = params; SPEED = speed_gbps;
    o_node* v = (o_node*)malloc(sizeof(o_node));
    if (!v) return -1;
    o_pod top;
    expand_pod(pod, &top);
    for (int n = 0; n < n_nodes; n++) {
        expand_node(&recs[n], v);
        reason[n] = (uint8_t)explain_one(v, &top, now);
    }
    free(v);
    return 0;
}
