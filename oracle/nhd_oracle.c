/*
 * nhd_oracle.c — ORACLE: a literal CPU restatement of the reference hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in nhd_b200/ (the product) may include,
 * link or call this file; only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs use it, as the checker or as the timed
 * CPU baseline.
 *
 * Parity pin: the reference's own tests hold no vectors for this path
 * (SURVEY.md section 4), so this restatement is pinned against the UNMODIFIED
 * reference modules imported in the build container — tests/test_oracle_vs_reference.py
 * (live, randomized) and the frozen vectors under tests/golden/ made by
 * tests/golden/make_golden.py.
 *
 * It consumes the same wire records as the product C-ABI (include/nhd_b200.h),
 * expands them into plain per-core / per-GPU / per-NIC lists shaped like the
 * reference's Node objects, and then follows the reference statement by
 * statement, deliberately WITHOUT any of the product's shortcuts: every
 * eligible node is evaluated for every pod, candidate lists are materialised,
 * and Python set semantics come from pyset_model.c.
 *
 * Reference functions restated (file:line in the reference checkout):
 *   NHDScheduler.InitialNodeFilter        nhd/NHDScheduler.py:235-247
 *   NHDScheduler.AttemptScheduling        nhd/NHDScheduler.py:277-304 (compute lines)
 *   Matcher.FindNode                      nhd/Matcher.py:27-63
 *   Matcher.FilterPodResources            nhd/Matcher.py:65-84
 *   Matcher.FilterNumaTopology            nhd/Matcher.py:86-280
 *   Matcher.IntersectResources            nhd/Matcher.py:283-391
 *   Matcher.SelectNode                    nhd/Matcher.py:393-421
 *   Matcher.GetNumaGroupIdx               nhd/Matcher.py:423-452
 *   Node.GetFreeCpuCores                  nhd/Node.py:250-264
 *   Node.GetFreeGPUPCICount               nhd/Node.py:266-273
 *   Node.GetNumaNICPCIResources           nhd/Node.py:275-281
 *   Node.GetFreeNumaNicResources          nhd/Node.py:283-296
 *   Node.GetFreeNumaGPUs                  nhd/Node.py:456-462
 *   Node.GetNextGpuFree                   nhd/Node.py:495-500
 *   Node.GetFreeCpuBatch                  nhd/Node.py:502-519
 *   Node.ClaimPodNICResources             nhd/Node.py:644-646
 *   Node.GetFreePciGpuFromNic             nhd/Node.py:648-655
 *   Node.GetNicObjFromIndex               nhd/Node.py:657-661
 *   Node.SetPhysicalIdsFromMapping        nhd/Node.py:663-841
 *   Node.SetBusy / IsBusy                 nhd/Node.py:843-850
 *   CfgTopology.GetTotal{Gpus,Cpus,NICs}Requested   nhd/CfgTopology.py:199-232
 */
#include "nhd_oracle.h"
#include "pyset_model.h"

#include <math.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------- */
/* Expanded node / pod model (shaped like nhd/Node.py and nhd/CfgTopology.py) */
/* ------------------------------------------------------------------------- */

typedef struct { int core, sibling, socket, used; } o_core;     /* NodeCore  Node.py:23-31  */
typedef struct { double speed; int numa_node, pciesw, pods_used, idx; } o_nic;  /* NodeNic :37-56 */
typedef struct { int numa_node, pciesw, used; } o_gpu;          /* NodeGpu   Node.py:74-83  */

typedef struct {
    int sockets, numa_nodes, smt_enabled, cores_per_proc;
    int n_cores;  o_core cores[NHD_MAX_LCORES];
    int n_gpus;   o_gpu  gpus[NHD_MAX_GPUS];
    int n_nics;   o_nic  nics[NHD_MAX_NICS];
    int free_hugepages_gb;
    int active, maintenance;
    uint64_t groups;
    double busy_time;
} o_node;

typedef struct {
    int n_gpus; int feeders[NHD_MAX_GROUP_GPUS];
    int n_proc, n_helpers, proc_smt, helper_smt, has_nic_cores;
    double rx, tx;
} o_group;

typedef struct {
    int n_groups; o_group g[NHD_MAX_GROUPS];
    int n_misc, misc_smt, hugepages_gb, map_type;
    uint64_t groups;
} o_pod;

typedef struct { uint8_t len; uint8_t v[7]; } otuple;
typedef struct { uint8_t numa[NHD_MAX_GROUPS]; uint8_t idx[NHD_MAX_GROUPS]; } onic;   /* [(numa, nic idx)] * G */

typedef struct {
    otuple* gpu; int n_gpu;      /* filts[0]['gpu'][n] */
    otuple* cpu; int n_cpu;      /* filts[0]['cpu'][n] */
    onic*   nic; int n_nic;      /* filts[0]['nic'][n] */
} o_filts;

static void filts_free(o_filts* f)
{
    free(f->gpu); free(f->cpu); free(f->nic);
    memset(f, 0, sizeof(*f));
}

static const nhd_oracle_params* P;   /* solver constants, set per call */
static const double* SPEED;          /* speed class -> NodeNic.speed */

/* ---- record <-> expanded node ------------------------------------------- */

static void expand_node(const nhd_node_rec* r, o_node* n)
{
    memset(n, 0, sizeof(*n));
    n->sockets = r->n_numa;
    n->numa_nodes = r->n_numa;                       /* Node.py:336 */
    n->smt_enabled = (r->flags & NHD_NODE_SMT) != 0;
    int cores = r->phys_cores;
    n->cores_per_proc = cores / n->sockets;          /* Node.py:338 */
    n->n_cores = n->smt_enabled ? cores * 2 : cores; /* Node.py:341 */
    for (int c = 0; c < n->n_cores; c++) {
        /* Node.py:344: int(int(c % cores) // (cores/self.sockets)), float floor-division */
        int proc = (int)floor((double)(c % cores) / ((double)cores / (double)n->sockets));
        int sib = n->smt_enabled ? (c < cores ? c + cores : c - cores) : -1;   /* :345-348 */
        n->cores[c].core = c;
        n->cores[c].socket = proc;
        n->cores[c].sibling = sib;
        n->cores[c].used = (int)((r->used[c >> 6] >> (c & 63)) & 1);
    }
    n->n_gpus = r->n_gpus;
    for (int i = 0; i < n->n_gpus; i++) {
        int numa = 0;
        for (int k = 0; k < NHD_MAX_NUMA; k++)
            if ((r->gpu_numa_mask[k] >> i) & 1) numa = k;
        n->gpus[i].numa_node = numa;
        n->gpus[i].pciesw = (int)((r->gpu_sw >> (4 * i)) & 0xF);
        n->gpus[i].used = (r->gpu_used >> i) & 1;
    }
    n->n_nics = r->n_nics;
    int nidx[NHD_MAX_NUMA] = {0};
    for (int i = 0; i < n->n_nics; i++) {
        int numa = 0;
        for (int k = 0; k < NHD_MAX_NUMA; k++)
            if ((r->nic_numa_mask[k] >> i) & 1) numa = k;
        n->nics[i].numa_node = numa;
        n->nics[i].pciesw = (int)((r->nic_sw[i >> 4] >> (4 * (i & 15))) & 0xF);
        n->nics[i].speed = SPEED[(r->nic_speed[i >> 4] >> (4 * (i & 15))) & 0xF];
        n->nics[i].pods_used = (r->nic_inuse >> i) & 1;
        n->nics[i].idx = nidx[numa]++;               /* Node.py:413-418 */
    }
    n->free_hugepages_gb = r->free_hugepages_gb;
    n->active = (r->flags & NHD_NODE_ACTIVE) != 0;
    n->maintenance = (r->flags & NHD_NODE_MAINTENANCE) != 0;
    n->groups = r->group_mask;
    n->busy_time = r->busy_time;
}

static void collapse_node(const o_node* n, nhd_node_rec* r)
{
    /* only the mutable fields change on this path */
    memset(r->used, 0, sizeof(r->used));
    for (int c = 0; c < n->n_cores; c++)
        if (n->cores[c].used) r->used[c >> 6] |= 1ULL << (c & 63);
    r->gpu_used = 0;
    for (int i = 0; i < n->n_gpus; i++)
        if (n->gpus[i].used) r->gpu_used |= (uint16_t)(1u << i);
    r->nic_inuse = 0;
    for (int i = 0; i < n->n_nics; i++)
        if (n->nics[i].pods_used > 0) r->nic_inuse |= 1u << i;
    r->free_hugepages_gb = n->free_hugepages_gb;
    r->busy_time = n->busy_time;
}

static void expand_pod(const nhd_pod* w, o_pod* p)
{
    memset(p, 0, sizeof(*p));
    p->n_groups = w->n_groups;
    for (int g = 0; g < w->n_groups; g++) {
        const nhd_pod_group* wg = &w->groups[g];
        o_group* og = &p->g[g];
        og->n_gpus = wg->n_gpus;
        for (int j = 0; j < wg->n_gpus; j++) og->feeders[j] = wg->gpu_feeders[j];
        og->n_proc = wg->n_proc;
        og->n_helpers = wg->n_helpers;
        og->proc_smt = (wg->flags & NHD_GRP_PROC_SMT) != 0;
        og->helper_smt = (wg->flags & NHD_GRP_HELPER_SMT) != 0;
        og->has_nic_cores = (wg->flags & NHD_GRP_HAS_NIC_CORES) != 0;
        og->rx = wg->rx_gbps;
        og->tx = wg->tx_gbps;
    }
    p->n_misc = w->n_misc;
    p->misc_smt = (w->flags & NHD_POD_MISC_SMT) != 0;
    p->hugepages_gb = w->hugepages_gb;
    p->map_type = w->map_type;
    p->groups = w->group_mask;
}

/* ---- Node queries -------------------------------------------------------- */

/* Node.IsBusy, Node.py:847-850 */
static int node_is_busy(const o_node* v, double now)
{
    double last_busy_time_seconds = now - v->busy_time;
    return last_busy_time_seconds < P->min_busy_secs;
}

/* Node.GetFreeNumaGPUs, Node.py:456-462 */
static void get_free_numa_gpus(const o_node* v, int* gfree)
{
    for (int k = 0; k < v->numa_nodes; k++) gfree[k] = 0;
    for (int i = 0; i < v->n_gpus; i++)
        if (!v->gpus[i].used) gfree[v->gpus[i].numa_node] += 1;
}

/* Node.GetFreeCpuCores, Node.py:250-264 */
static void get_free_cpu_cores(const o_node* v, int* fl)
{
    for (int k = 0; k < v->numa_nodes; k++) fl[k] = 0;
    for (int c = 0; c < v->cores_per_proc * v->sockets; c++) {
        if (!v->cores[c].used) {
            if (!v->smt_enabled)
                fl[v->cores[c].socket] += 1;
            else if (!v->cores[v->cores[c].sibling].used)
                fl[v->cores[c].socket] += 1;
        }
    }
}

/* Node.GetFreeNumaNicResources, Node.py:283-296 (sharing disabled branch) */
static void get_free_numa_nic_resources(const o_node* v, double ninfo[NHD_MAX_NUMA][NHD_MAX_NICS][2], int* cnt)
{
    for (int k = 0; k < v->numa_nodes; k++) cnt[k] = 0;
    for (int i = 0; i < v->n_nics; i++) {
        const o_nic* n = &v->nics[i];
        double f = (n->pods_used > 0) ? 0.0 : n->speed * P->nic_bw_avail_percent;
        ninfo[n->numa_node][cnt[n->numa_node]][0] = f;
        ninfo[n->numa_node][cnt[n->numa_node]][1] = f;
        cnt[n->numa_node]++;
    }
}

/* Node.GetFreeGPUPCICount, Node.py:266-273: defaultdict switch -> free GPUs */
static void get_free_gpu_pci_count(const o_node* v, int* ginfo /* [NHD_MAX_SWITCHES] */)
{
    for (int s = 0; s < NHD_MAX_SWITCHES; s++) ginfo[s] = 0;
    for (int i = 0; i < v->n_gpus; i++)
        if (!v->gpus[i].used) ginfo[v->gpus[i].pciesw] += 1;
}

/* Node.GetNumaNICPCIResources, Node.py:275-281: ninfo[numa][idx] = pciesw */
static void get_numa_nic_pci_resources(const o_node* v, int ninfo[NHD_MAX_NUMA][NHD_MAX_NICS])
{
    for (int i = 0; i < v->n_nics; i++)
        ninfo[v->nics[i].numa_node][v->nics[i].idx] = v->nics[i].pciesw;
}

/* ---- itertools.product(range(k), repeat=len): odometer, last digit fastest -- */
static int product_next(uint8_t* p, int len, int k)
{
    for (int i = len - 1; i >= 0; i--) {
        if (p[i] + 1 < k) { p[i]++; return 1; }
        p[i] = 0;
    }
    return 0;
}

static uint64_t tuple_key(const otuple* t)
{
    int items[8];
    for (int i = 0; i < t->len; i++) items[i] = t->v[i];
    return pyset_tuple_key(items, t->len);
}

static uint64_t tuple_hash(const otuple* t)
{
    int items[8];
    for (int i = 0; i < t->len; i++) items[i] = t->v[i];
    return py_hash_tuple(items, t->len);
}

static otuple key_to_tuple(uint64_t key)
{
    int items[8], len;
    otuple t; memset(&t, 0, sizeof(t));
    pyset_key_tuple(key, items, &len);
    t.len = (uint8_t)len;
    for (int i = 0; i < len; i++) t.v[i] = (uint8_t)items[i];
    return t;
}

static int tuple_eq(const otuple* a, const otuple* b)
{
    return a->len == b->len && memcmp(a->v, b->v, a->len) == 0;
}

/* list(set) -> freshly malloc'd tuple array */
static otuple* set_to_tuple_list(const pyset* s, int* n_out)
{
    uint64_t* keys = (uint64_t*)malloc(sizeof(uint64_t) * (s->used + 1));
    size_t n = pyset_list(s, keys, NULL);
    otuple* out = (otuple*)malloc(sizeof(otuple) * (n + 1));
    for (size_t i = 0; i < n; i++) out[i] = key_to_tuple(keys[i]);
    free(keys);
    *n_out = (int)n;
    return out;
}

static pyset* new_set(void)
{
    pyset* s = (pyset*)malloc(sizeof(pyset));
    pyset_init(s);
    return s;
}

/* ------------------------------------------------------------------------- */
/* Matcher.FilterNumaTopology, one node at a time (Matcher.py:86-280).        */
/* The reference runs the three stages node-list-major; the stages of         */
/* different nodes are independent, so evaluating them node by node yields    */
/* the same filts / cand_nodes.                                               */
/* ------------------------------------------------------------------------- */

/* GPU stage, Matcher.py:95-149.  Returns 0 when the node is dropped. */
static int filter_gpu_stage(const o_node* v, const o_pod* top, double now, o_filts* f)
{
    int G = top->n_groups;
    int req_gpus[NHD_MAX_GROUPS], sum = 0;                 /* CfgTopology.py:199-200 */
    for (int g = 0; g < G; g++) { req_gpus[g] = top->g[g].n_gpus; sum += req_gpus[g]; }

    if (sum > 0)                                           /* :107-111 */
        if (node_is_busy(v, now))
            return 0;

    pyset* stmp = new_set();
    int free_gpus[NHD_MAX_NUMA];
    get_free_numa_gpus(v, free_gpus);                      /* :115 */

    otuple p; memset(&p, 0, sizeof(p)); p.len = (uint8_t)G;
    do {                                                   /* :118-129 */
        int ttl[NHD_MAX_NUMA] = {0};
        for (int idx = 0; idx < G; idx++) ttl[p.v[idx]] += req_gpus[idx];
        int ok = 1;
        for (int x = 0; x < v->numa_nodes; x++) if (!(ttl[x] <= free_gpus[x])) ok = 0;
        if (ok) pyset_add(stmp, tuple_key(&p), tuple_hash(&p));
    } while (product_next(p.v, G, v->numa_nodes));

    int keep = stmp->used != 0;                            /* :132-136 */
    f->gpu = set_to_tuple_list(stmp, &f->n_gpu);           /* :141 (done even when dropped) */
    free(stmp);
    return keep;
}

/* CPU stage, Matcher.py:152-222 */
static int filter_cpu_stage(const o_node* v, const o_pod* top, o_filts* f)
{
    int G = top->n_groups;
    int fcpu[NHD_MAX_NUMA];
    get_free_cpu_cores(v, fcpu);                           /* :164 */

    int clist[NHD_MAX_GROUPS + 1], nc = 0;
    for (int g = 0; g < G; g++) {                          /* :179-194, CfgTopology.py:202-217 */
        const o_group* t = &top->g[g];
        int t00 = t->n_proc;
        for (int j = 0; j < t->n_gpus; j++) t00 += t->feeders[j];
        int t10 = t->n_helpers;
        if (v->smt_enabled) {
            int tot = 0;
            if (t->proc_smt) tot += (int)ceil(t00 / 2.0); else tot += t00;
            if (t->helper_smt) tot += (int)ceil(t10 / 2.0); else tot += t10;
            clist[nc++] = tot;
        } else {
            clist[nc++] = t00 + t10;
        }
    }
    /* :197-201 — `if req_cpus['misc'][1]` tests an Enum member, which is always
     * truthy, so SMT nodes halve the misc cores whatever misc_cores_smt says. */
    if (v->smt_enabled)
        clist[nc++] = (int)ceil(top->n_misc / 2.0);
    else
        clist[nc++] = top->n_misc;

    pyset* stmp = new_set();
    otuple p; memset(&p, 0, sizeof(p)); p.len = (uint8_t)nc;
    do {                                                   /* :203-212 */
        int ttl[NHD_MAX_NUMA] = {0};
        for (int idx = 0; idx < nc; idx++) ttl[p.v[idx]] += clist[idx];
        int ok = 1;
        for (int x = 0; x < v->numa_nodes; x++) if (!(ttl[x] <= fcpu[x])) ok = 0;
        if (ok) pyset_add(stmp, tuple_key(&p), tuple_hash(&p));
    } while (product_next(p.v, nc, v->numa_nodes));

    int keep = stmp->used != 0;                            /* :214-218 */
    f->cpu = set_to_tuple_list(stmp, &f->n_cpu);           /* :220 */
    free(stmp);
    return keep;
}

/* NIC stage, Matcher.py:224-276 */
static int filter_nic_stage(const o_node* v, const o_pod* top, o_filts* f)
{
    int G = top->n_groups;
    int K = v->numa_nodes;
    double req_nics[NHD_MAX_GROUPS][2];                    /* CfgTopology.py:219-232 */
    for (int g = 0; g < G; g++) { req_nics[g][0] = top->g[g].rx; req_nics[g][1] = top->g[g].tx; }

    static _Thread_local double nnic_free[NHD_MAX_NUMA][NHD_MAX_NICS][2];
    int ncnt[NHD_MAX_NUMA];
    get_free_numa_nic_resources(v, nnic_free, ncnt);       /* :240 */

    int cap = 64;
    f->nic = (onic*)malloc(sizeof(onic) * cap);
    f->n_nic = 0;

    uint8_t p[NHD_MAX_GROUPS] = {0};
    do {                                                   /* :242-243 */
        /* :245-247 groups on each NUMA node, and the size of product(range(n), repeat=len) */
        int nidx_len[NHD_MAX_NUMA];
        long combos[NHD_MAX_NUMA];
        for (int numa = 0; numa < K; numa++) {
            int len = 0;
            for (int i = 0; i < G; i++) if (p[i] == numa) len++;
            nidx_len[numa] = len;
            long c = 1;
            for (int i = 0; i < len; i++) c *= ncnt[numa];
            combos[numa] = c;                              /* len(nic_combos[numa]) */
        }
        /* :250 idx_combos = product(*[range(len(x)) for x in nic_combos]), last NUMA fastest */
        int empty = 0;
        for (int numa = 0; numa < K; numa++) if (combos[numa] == 0) empty = 1;
        if (!empty) {
            long combo_idx[NHD_MAX_NUMA] = {0};
            for (;;) {
                /* :253-256: c[numaidx] = list(nic_combos[numaidx][numa_combo_idx[numaidx]]) */
                uint8_t c[NHD_MAX_NUMA][NHD_MAX_GROUPS];
                int cpos[NHD_MAX_NUMA] = {0};
                for (int numa = 0; numa < K; numa++) {
                    long r = combo_idx[numa];
                    for (int i = nidx_len[numa] - 1; i >= 0; i--) {     /* tuple #r of the product */
                        c[numa][i] = (uint8_t)(r % ncnt[numa]);
                        r /= ncnt[numa];
                    }
                }
                /* :254 nic_ttls = copy.deepcopy(nnic_free[n]) */
                static _Thread_local double nic_ttls[NHD_MAX_NUMA][NHD_MAX_NICS][2];
                memcpy(nic_ttls, nnic_free, sizeof(nic_ttls));
                /* :258 ttl_list = [c[np].pop(0) for np in p] */
                uint8_t ttl_list[NHD_MAX_GROUPS];
                for (int g = 0; g < G; g++) ttl_list[g] = c[p[g]][cpos[p[g]]++];
                /* :261-263 */
                for (int xi = 0; xi < G; xi++) {
                    nic_ttls[p[xi]][ttl_list[xi]][0] -= req_nics[xi][0];
                    nic_ttls[p[xi]][ttl_list[xi]][1] -= req_nics[xi][1];
                }
                /* :267 */
                int any_neg = 0;
                for (int y = 0; y < K; y++)
                    for (int z = 0; z < ncnt[y]; z++)
                        for (int x = 0; x < 2; x++)
                            if (nic_ttls[y][z][x] < 0) any_neg = 1;
                if (!any_neg) {                            /* :268 */
                    if (f->n_nic == cap) { cap *= 2; f->nic = (onic*)realloc(f->nic, sizeof(onic) * cap); }
                    onic* e = &f->nic[f->n_nic++];
                    memset(e, 0, sizeof(*e));
                    for (int g = 0; g < G; g++) { e->numa[g] = p[g]; e->idx[g] = ttl_list[g]; }
                }
                /* advance idx_combos */
                int k = K - 1;
                for (; k >= 0; k--) {
                    if (combo_idx[k] + 1 < combos[k]) { combo_idx[k]++; break; }
                    combo_idx[k] = 0;
                }
                if (k < 0) break;
            }
        }
    } while (product_next(p, G, K));

    return f->n_nic != 0;                                  /* :270-274 */
}

/* ------------------------------------------------------------------------- */
/* Matcher.IntersectResources for one candidate node (Matcher.py:283-391).    */
/* Returns 0 when the node is removed from filts[1].                           */
/* ------------------------------------------------------------------------- */
static int intersect_node(const o_node* v, const o_pod* top, o_filts* f)
{
    int G = top->n_groups;

    if (top->map_type == NHD_MAP_PCI) {                    /* :295-335 */
        int gsw[NHD_MAX_SWITCHES];
        static _Thread_local int nsw[NHD_MAX_NUMA][NHD_MAX_NICS];
        get_free_gpu_pci_count(v, gsw);                    /* :307 */
        get_numa_nic_pci_resources(v, nsw);                /* :308 */
        int* to_remove = (int*)calloc((size_t)f->n_nic + 1, sizeof(int));
        int n_remove = 0;
        for (int e = 0; e < f->n_nic; e++) {               /* :312-322 */
            int nicswcount[NHD_MAX_SWITCHES] = {0};
            for (int g = 0; g < G; g++)
                nicswcount[nsw[f->nic[e].numa[g]][f->nic[e].idx[g]]] += 1;
            for (int s = 0; s < NHD_MAX_SWITCHES; s++)
                if (nicswcount[s] > 0 && gsw[s] < nicswcount[s]) { to_remove[e] = 1; n_remove++; }
        }
        if (n_remove != 0) {                               /* :325-335: delete each listed entry (once) */
            int w = 0;
            for (int e = 0; e < f->n_nic; e++)
                if (!to_remove[e]) f->nic[w++] = f->nic[e];
            f->n_nic = w;
        }
        free(to_remove);
    }

    /* :344-349 */
    pyset* sg = new_set(); pyset* sc = new_set(); pyset* sn = new_set();
    pyset* t1 = new_set(); pyset* isect = new_set();
    for (int i = 0; i < f->n_gpu; i++)                     /* set(gpu_tuples) */
        pyset_add(sg, tuple_key(&f->gpu[i]), tuple_hash(&f->gpu[i]));
    for (int i = 0; i < f->n_cpu; i++) {                   /* set([x[:-1] ...]) */
        otuple t = f->cpu[i]; t.len--; t.v[t.len] = 0;
        pyset_add(sc, tuple_key(&t), tuple_hash(&t));
    }
    for (int i = 0; i < f->n_nic; i++) {                   /* set([list(zip(*x))[0] ...]) */
        otuple t; memset(&t, 0, sizeof(t)); t.len = (uint8_t)G;
        for (int g = 0; g < G; g++) t.v[g] = f->nic[i].numa[g];
        pyset_add(sn, tuple_key(&t), tuple_hash(&t));
    }
    pyset_intersection(sg, sc, t1);
    pyset_intersection(t1, sn, isect);
    int n_isect;
    otuple* intersect = set_to_tuple_list(isect, &n_isect);

    int keep = 1;
    if (n_isect == 0) {                                    /* :352-359 */
        keep = 0;
    } else {
        /* :365-368 diff = set(gpu) - set(intersect) */
        int diff = 0;
        for (int i = 0; i < f->n_gpu; i++) {
            int found = 0;
            for (int j = 0; j < n_isect; j++) if (tuple_eq(&f->gpu[i], &intersect[j])) found = 1;
            if (!found) diff++;
        }
        if (diff) {
            free(f->gpu);
            f->gpu = (otuple*)malloc(sizeof(otuple) * (size_t)n_isect);
            memcpy(f->gpu, intersect, sizeof(otuple) * (size_t)n_isect);
            f->n_gpu = n_isect;
        }
        /* :371-374 `for c in list: if ...: list.remove(c)` — mutation while iterating */
        for (int i = 0; i < f->n_cpu; i++) {
            otuple t = f->cpu[i]; t.len--;
            int in = 0;
            for (int j = 0; j < n_isect; j++) if (tuple_eq(&t, &intersect[j])) in = 1;
            if (!in) {
                memmove(&f->cpu[i], &f->cpu[i + 1], sizeof(otuple) * (size_t)(f->n_cpu - i - 1));
                f->n_cpu--;
                /* the list iterator still advances: the element that slid into slot i is skipped */
            }
        }
        /* :378-382 same pattern with enumerate + del */
        for (int i = 0; i < f->n_nic; i++) {
            otuple t; memset(&t, 0, sizeof(t)); t.len = (uint8_t)G;
            for (int g = 0; g < G; g++) t.v[g] = f->nic[i].numa[g];
            int in = 0;
            for (int j = 0; j < n_isect; j++) if (tuple_eq(&t, &intersect[j])) in = 1;
            if (!in) {
                memmove(&f->nic[i], &f->nic[i + 1], sizeof(onic) * (size_t)(f->n_nic - i - 1));
                f->n_nic--;
            }
        }
        /* :384-389: all three lists are non-empty here (each keeps its entries that match
         * an intersection member), so the `del filts[1][n]` branch is unreachable. */
    }
    free(intersect);
    free(sg); free(sc); free(sn); free(t1); free(isect);
    return keep;
}

/* Matcher.GetNumaGroupIdx, Matcher.py:423-452 */
typedef struct { otuple gpu; otuple cpu; onic nic; } o_mapping;

static int get_numa_group_idx(int numa_nodes, const o_filts* f, int G, o_mapping* m)
{
    int gidx = 0, gval = -1;
    for (int x = 0; x < f->n_gpu; x++) {                   /* :428-437 */
        int mx = -1, mn = 1 << 30;
        for (int y = 0; y < numa_nodes; y++) {
            int cnt = 0;
            for (int i = 0; i < f->gpu[x].len; i++) if (f->gpu[x].v[i] == y) cnt++;
            if (cnt > mx) mx = cnt;
            if (cnt < mn) mn = cnt;
        }
        int d = mx - mn;
        if (x == 0) { gidx = 0; gval = d; }
        else if (d > gval) { gidx = x; gval = d; }
    }
    m->gpu = f->gpu[gidx];                                 /* :439 */
    int cidx = -1;                                         /* :442-444 */
    for (int i = 0; i < f->n_cpu; i++) {
        otuple t = f->cpu[i]; t.len--;
        if (tuple_eq(&t, &m->gpu)) { cidx = i; break; }
    }
    if (cidx < 0) return -1;
    m->cpu = f->cpu[cidx];
    int nidx = -1;                                         /* :447-449 */
    for (int i = 0; i < f->n_nic; i++) {
        int eq = 1;
        for (int g = 0; g < G; g++) if (f->nic[i].numa[g] != m->gpu.v[g]) eq = 0;
        if (eq) { nidx = i; break; }
    }
    if (nidx < 0) return -1;
    m->nic = f->nic[nidx];
    return 0;
}

/* One node through FilterPodResources + the three filter stages + intersection.
 * Returns 1 if the node ends up in filts[1]; its final filts are left in *f. */
static int evaluate_node(const o_node* v, const o_pod* top, double now, o_filts* f)
{
    memset(f, 0, sizeof(*f));
    if (v->maintenance) return 0;                          /* Matcher.py:73 */
    if (top->hugepages_gb > v->free_hugepages_gb) return 0;/* :78 */
    if (!filter_gpu_stage(v, top, now, f)) return 0;
    if (!filter_cpu_stage(v, top, f)) return 0;
    if (!filter_nic_stage(v, top, f)) return 0;
    if (!intersect_node(v, top, f)) return 0;
    return 1;
}

/* ------------------------------------------------------------------------- */
/* Node.GetFreeCpuBatch, Node.py:502-519                                      */
/* ------------------------------------------------------------------------- */
static int get_free_cpu_batch(const o_node* v, int numa, int num, int smt, int* cpus)
{
    int n = 0;
    for (int ci = 0; ci < v->n_cores; ci++) {
        const o_core* c = &v->cores[ci];
        if (num == 0) break;
        if (c->socket == numa && !c->used) {
            if (v->smt_enabled) {
                if (!v->cores[c->sibling].used) {
                    if (smt && num >= 2) {
                        cpus[n++] = c->core; cpus[n++] = c->sibling;
                        num -= 2;
                    } else {
                        cpus[n++] = c->core;
                        num -= 1;
                    }
                }
            } else {
                cpus[n++] = c->core;
                num -= 1;
            }
        }
    }
    return n;
}

/* Node.SetPhysicalIdsFromMapping, Node.py:663-841.  Returns the binding status. */
static int set_physical_ids_from_mapping(o_node* v, const o_mapping* mapping, const o_pod* top, nhd_binding* b)
{
    int used_cpus[NHD_MAX_LCORES * 2], n_used_cpus = 0;
    int used_gpus[NHD_MAX_POD_GPUS + 1], n_used_gpus = 0;
    int used_nics[NHD_MAX_GROUPS], n_used_nics = 0;         /* NIC list index per group that recorded speed */
    int out_cores = 0, out_gpus = 0;
    int group_cpus[NHD_MAX_LCORES * 2];
    int G = top->n_groups;

    for (int pi = 0; pi < G; pi++) {                       /* :674 */
        const o_group* pv = &top->g[pi];
        int group_numa_node = mapping->gpu.v[pi];          /* :679 */
        int cidx = 0;
        int gcpu_req = pv->n_proc;                         /* :681 */
        for (int j = 0; j < pv->n_gpus; j++) gcpu_req += pv->feeders[j];
        int n_group_cpus = get_free_cpu_batch(v, group_numa_node, gcpu_req, pv->proc_smt, group_cpus);   /* :682 */
        if (n_group_cpus != gcpu_req) goto index_error;    /* :685-687 */

        /* :701-705 GetNicObjFromIndex */
        int nobj = -1;
        for (int ni = 0; ni < v->n_nics; ni++)
            if (mapping->nic.idx[pi] == v->nics[ni].idx && v->nics[ni].numa_node == mapping->nic.numa[pi]) { nobj = ni; break; }
        if (nobj < 0) goto index_error;
        b->nic_list_index[pi] = (uint8_t)nobj;

        for (int gi = 0; gi < pv->n_gpus; gi++) {          /* :707 */
            int gdev = -1;
            for (int x = 0; x < v->n_gpus; x++)            /* GetFreePciGpuFromNic :648-655 */
                if (v->gpus[x].pciesw == v->nics[nobj].pciesw && !v->gpus[x].used) { gdev = x; break; }
            if (gdev < 0) {
                if (top->map_type == NHD_MAP_PCI) goto index_error;        /* :711-713 */
                for (int x = 0; x < v->n_gpus; x++)        /* GetNextGpuFree :495-500 */
                    if (v->gpus[x].numa_node == group_numa_node && !v->gpus[x].used) { gdev = x; break; }
            }
            if (gdev < 0) goto index_error;                /* :718-720 */
            v->gpus[gdev].used = 1;                        /* :724-726 */
            used_gpus[n_used_gpus++] = gdev;
            if (out_gpus < NHD_MAX_POD_GPUS) b->gpu_index[out_gpus++] = (uint8_t)gdev;
            for (int k = 0; k < pv->feeders[gi]; k++) {    /* :728-732 */
                int core = group_cpus[cidx];
                v->cores[core].used = 1;
                used_cpus[n_used_cpus++] = core;
                if (out_cores < NHD_MAX_POD_CORES) b->cores[out_cores++] = (uint8_t)core;
                cidx++;
            }
        }
        for (int k = 0; k < pv->n_proc; k++) {             /* :735-739 */
            int core = group_cpus[cidx];
            v->cores[core].used = 1;
            used_cpus[n_used_cpus++] = core;
            if (out_cores < NHD_MAX_POD_CORES) b->cores[out_cores++] = (uint8_t)core;
            cidx++;
        }
        if (pv->has_nic_cores)                             /* :742-755 (speed_used stays with the caller) */
            used_nics[n_used_nics++] = nobj;
        if (cidx != n_group_cpus) goto index_error;        /* :767-769 */

        int helper_req[NHD_MAX_LCORES * 2];                /* :773-788 */
        int n_helper = get_free_cpu_batch(v, group_numa_node, pv->n_helpers, pv->helper_smt, helper_req);
        if (pv->n_helpers != n_helper) goto index_error;
        for (int k = 0; k < pv->n_helpers; k++) {
            int core = helper_req[k];
            v->cores[core].used = 1;
            used_cpus[n_used_cpus++] = core;
            if (out_cores < NHD_MAX_POD_CORES) b->cores[out_cores++] = (uint8_t)core;
        }
    }

    if (top->hugepages_gb > 0)                             /* :794-796 */
        v->free_hugepages_gb -= top->hugepages_gb;

    {                                                      /* :799-815 */
        int misc_cpus[NHD_MAX_LCORES * 2];
        int n_misc = get_free_cpu_batch(v, mapping->cpu.v[mapping->cpu.len - 1], top->n_misc, top->misc_smt, misc_cpus);
        if (top->n_misc != n_misc) goto index_error;
        for (int k = 0; k < top->n_misc; k++) {
            int core = misc_cpus[k];
            v->cores[core].used = 1;
            used_cpus[n_used_cpus++] = core;
            if (out_cores < NHD_MAX_POD_CORES) b->cores[out_cores++] = (uint8_t)core;
        }
    }
    b->n_cores = (uint8_t)out_cores;
    b->n_gpus = (uint8_t)out_gpus;

    /* NHDScheduler.py:302-304: nidx = list({x[0] for x in nic_list}); ClaimPodNICResources */
    {
        pyset* s = new_set();
        for (int i = 0; i < n_used_nics; i++) pyset_add(s, (uint64_t)used_nics[i], py_hash_int(used_nics[i]));
        uint64_t keys[NHD_MAX_GROUPS + 1];
        size_t n = pyset_list(s, keys, NULL);
        free(s);
        b->n_claimed = (uint8_t)n;
        for (size_t i = 0; i < n; i++) {
            b->claimed_nics[i] = (uint8_t)keys[i];
            v->nics[keys[i]].pods_used += 1;               /* Node.py:644-646 */
        }
    }
    return NHD_PLACED;

index_error:                                               /* :825-837 */
    for (int i = 0; i < n_used_cpus; i++) v->cores[used_cpus[i]].used = 0;
    for (int i = 0; i < n_used_gpus; i++) v->gpus[used_gpus[i]].used = 0;   /* self.gpus[device_id]: ids are list indices by contract */
    /* The hugepages decrement (:794-796) precedes the misc-core batch; if that batch raised,
     * the reference would NOT restore hugepages.  That raise is unreachable after a
     * successful filter (DESIGN.md), so no rollback is modelled either. */
    b->n_cores = 0; b->n_gpus = 0; b->n_claimed = 0;
    memset(b->cores, 0, sizeof(b->cores));                 /* nothing stays assigned after the unwind */
    memset(b->gpu_index, 0, sizeof(b->gpu_index));
    /* :831-835 indexes self.nics by a *speed*: IndexError or TypeError when any NIC speed
     * was recorded before the failure. */
    return n_used_nics ? NHD_REF_WOULD_CRASH : NHD_ASSIGN_FAILED;
}

/* ------------------------------------------------------------------------- */
/* One pod: InitialNodeFilter + FindNode + SetBusy + assignment + claim       */
/* ------------------------------------------------------------------------- */
/* What the node loop of FindNode leaves behind for SelectNode: the first candidate and the first
 * candidate without GPUs, each with its filts (Matcher.py:55, 412-421).  The reference walks ALL
 * nodes for every pod; scan_range() does the same over [lo, hi) so that the walk can be split into
 * ranges (nhd_oracle_solve_mt) — node evaluations within one pod are independent of each other. */
typedef struct {
    int first_cand, first_nogpu;
    o_filts f_first, f_nogpu;
} scan_res;

static void scan_range(const o_node* nodes, int lo, int hi, const o_pod* top, double now,
                       scan_res* r, uint8_t* cand_out)
{
    r->first_cand = r->first_nogpu = -1;
    memset(&r->f_first, 0, sizeof(r->f_first)); memset(&r->f_nogpu, 0, sizeof(r->f_nogpu));
    for (int n = lo; n < hi; n++) {
        const o_node* v = &nodes[n];
        if (cand_out) cand_out[n] = 0;
        /* InitialNodeFilter, NHDScheduler.py:241-243 */
        if ((v->groups & top->groups) == 0) continue;
        if (!v->active) continue;
        o_filts f;
        int cand = evaluate_node(v, top, now, &f);
        if (cand && cand_out) cand_out[n] = 1;
        if (cand && r->first_cand < 0) {
            r->first_cand = n; r->f_first = f; memset(&f, 0, sizeof(f));
            if (v->n_gpus == 0) r->first_nogpu = n;        /* shares f_first */
        } else if (cand && r->first_nogpu < 0 && v->n_gpus == 0) {
            r->first_nogpu = n; r->f_nogpu = f; memset(&f, 0, sizeof(f));
        }
        filts_free(&f);
    }
}

static void scan_res_free(scan_res* r) { filts_free(&r->f_first); filts_free(&r->f_nogpu); }

/* Ranges in ascending node order -> the result of one walk over all of them. */
static void scan_merge(scan_res* parts, int n_parts, scan_res* out)
{
    out->first_cand = out->first_nogpu = -1;
    memset(&out->f_first, 0, sizeof(out->f_first)); memset(&out->f_nogpu, 0, sizeof(out->f_nogpu));
    for (int p = 0; p < n_parts; p++) {
        scan_res* r = &parts[p];
        int took_first = 0;
        if (r->first_cand >= 0 && out->first_cand < 0) {
            out->first_cand = r->first_cand;
            out->f_first = r->f_first; memset(&r->f_first, 0, sizeof(r->f_first));
            took_first = 1;
        }
        if (r->first_nogpu >= 0 && out->first_nogpu < 0) {
            out->first_nogpu = r->first_nogpu;
            if (r->first_nogpu == r->first_cand) {
                /* the range's first candidate has no GPUs: one filts for both roles; it is already
                 * out->f_first if this range supplied the overall first candidate */
                if (!took_first) { out->f_nogpu = r->f_first; memset(&r->f_first, 0, sizeof(r->f_first)); }
            } else {
                out->f_nogpu = r->f_nogpu; memset(&r->f_nogpu, 0, sizeof(r->f_nogpu));
            }
        }
        scan_res_free(r);
    }
}

static void finish_scheduling(o_node* nodes, const o_pod* top, double now, nhd_binding* b, scan_res* sr);

static void attempt_scheduling(o_node* nodes, int n_nodes, const o_pod* top, double now,
                               nhd_binding* b, uint8_t* cand_out)
{
    memset(b, 0, sizeof(*b));
    b->node = -1;
    b->n_groups = (uint8_t)top->n_groups;

    if (top->map_type != NHD_MAP_NUMA && top->map_type != NHD_MAP_PCI) {   /* Matcher.py:45-47 */
        b->status = NHD_BAD_MAP_TYPE;
        return;
    }
    scan_res sr;
    scan_range(nodes, 0, n_nodes, top, now, &sr, cand_out);
    finish_scheduling(nodes, top, now, b, &sr);
}

/* SelectNode, GetNumaGroupIdx, SetBusy, SetPhysicalIdsFromMapping on the walk's result. */
static void finish_scheduling(o_node* nodes, const o_pod* top, double now, nhd_binding* b, scan_res* sr)
{
    /* SelectNode inputs, Matcher.py:406-410 */
    int needsGpu = 0;
    for (int g = 0; g < top->n_groups; g++) if (top->g[g].n_gpus > 0) needsGpu = 1;
    const int first_cand = sr->first_cand, first_nogpu = sr->first_nogpu;
#define f_first (sr->f_first)
#define f_nogpu (sr->f_nogpu)

    if (first_cand < 0) {                                  /* Matcher.py:50-52 / 58-60 */
        b->status = NHD_NO_CANDIDATE;
        return;
    }

    /* SelectNode, Matcher.py:412-421 */
    int node = first_cand;
    const o_filts* f = &f_first;
    if (!needsGpu && first_nogpu >= 0) {
        node = first_nogpu;
        f = (first_nogpu == first_cand) ? &f_first : &f_nogpu;
    }

    o_mapping m;
    if (get_numa_group_idx(nodes[node].numa_nodes, f, top->n_groups, &m) != 0) {
        fprintf(stderr, "nhd_oracle: internal error: no matching cpu/nic tuple\n");
        abort();
    }
    b->node = node;
    for (int g = 0; g < top->n_groups; g++) {
        b->gpu_numa[g] = m.gpu.v[g];
        b->nic_numa[g] = m.nic.numa[g];
        b->nic_idx[g] = m.nic.idx[g];
    }
    for (int g = 0; g < m.cpu.len; g++) b->cpu_numa[g] = m.cpu.v[g];
    /* nic_list_index is a pure function of the mapping (GetNicObjFromIndex, Node.py:657-661):
     * report it for every group, also when the assignment later fails part-way */
    for (int g = 0; g < top->n_groups; g++)
        for (int ni = 0; ni < nodes[node].n_nics; ni++)
            if (m.nic.idx[g] == nodes[node].nics[ni].idx && nodes[node].nics[ni].numa_node == m.nic.numa[g]) {
                b->nic_list_index[g] = (uint8_t)ni;
                break;
            }

    nodes[node].busy_time = now;                           /* NHDScheduler.py:289, Node.py:843-845 */
    b->status = set_physical_ids_from_mapping(&nodes[node], &m, top, b);

    filts_free(&f_first); filts_free(&f_nogpu);
#undef f_first
#undef f_nogpu
}

/* ------------------------------------------------------------------------- */
/* public entry points                                                        */
/* ------------------------------------------------------------------------- */

void nhd_oracle_default_params(nhd_oracle_params* p)
{
    p->nic_bw_avail_percent = 0.9;   /* Node.py:18 */
    p->min_busy_secs = 30.0;         /* Node.py:107 */
}

int nhd_oracle_solve(const nhd_oracle_params* params, const double* speed_gbps,
                     int n_nodes, nhd_node_rec* recs,
                     int n_pods, const nhd_pod* pods, const double* now,
                     nhd_binding* out)
{
    P = params; SPEED = speed_gbps;
    o_node* nodes = (o_node*)malloc(sizeof(o_node) * (size_t)(n_nodes > 0 ? n_nodes : 1));
    if (!nodes) return -1;
    for (int n = 0; n < n_nodes; n++) expand_node(&recs[n], &nodes[n]);
    for (int i = 0; i < n_pods; i++) {
        o_pod top;
        expand_pod(&pods[i], &top);
        attempt_scheduling(nodes, n_nodes, &top, now[i], &out[i], NULL);
        if (out[i].node >= 0)
            collapse_node(&nodes[out[i].node], &recs[out[i].node]);
    }
    free(nodes);
    return 0;
}

/* ---- the same, with the per-pod walk over the nodes split over threads ---------------------- */
typedef struct {
    int T;
    pthread_barrier_t start, done;
    volatile int quit;
    const o_node* nodes; int n_nodes;
    const o_pod* top; double now;
    scan_res* parts;
} scan_pool;

typedef struct { scan_pool* pool; int t; } scan_worker;

static void pool_do_range(scan_pool* pl, int t)
{
    const long n = pl->n_nodes;
    scan_range(pl->nodes, (int)(n * t / pl->T), (int)(n * (t + 1) / pl->T), pl->top, pl->now, &pl->parts[t], NULL);
}

static void* pool_main(void* arg)
{
    scan_worker* w = (scan_worker*)arg;
    for (;;) {
        pthread_barrier_wait(&w->pool->start);
        if (w->pool->quit) break;
        pool_do_range(w->pool, w->t);
        pthread_barrier_wait(&w->pool->done);
    }
    return NULL;
}

int nhd_oracle_solve_mt(const nhd_oracle_params* params, const double* speed_gbps,
                        int n_nodes, nhd_node_rec* recs,
                        int n_pods, const nhd_pod* pods, const double* now,
                        nhd_binding* out, int n_threads)
{
    if (n_threads < 2)
        return nhd_oracle_solve(params, speed_gbps, n_nodes, recs, n_pods, pods, now, out);
    P = params; SPEED = speed_gbps;
    o_node* nodes = (o_node*)malloc(sizeof(o_node) * (size_t)(n_nodes > 0 ? n_nodes : 1));
    if (!nodes) return -1;
    for (int n = 0; n < n_nodes; n++) expand_node(&recs[n], &nodes[n]);

    scan_pool pl;
    memset(&pl, 0, sizeof(pl));
    pl.T = n_threads; pl.nodes = nodes; pl.n_nodes = n_nodes;
    pl.parts = (scan_res*)calloc((size_t)n_threads, sizeof(scan_res));
    pthread_t* th = (pthread_t*)calloc((size_t)n_threads, sizeof(pthread_t));
    scan_worker* ws = (scan_worker*)calloc((size_t)n_threads, sizeof(scan_worker));
    if (!pl.parts || !th || !ws) return -1;
    pthread_barrier_init(&pl.start, NULL, (unsigned)n_threads);
    pthread_barrier_init(&pl.done, NULL, (unsigned)n_threads);
    int started = 1;
    for (int t = 1; t < n_threads; t++) {
        ws[t].pool = &pl; ws[t].t = t;
        if (pthread_create(&th[t], NULL, pool_main, &ws[t]) != 0) break;
        started++;
    }
    if (started != n_threads) {                  /* could not get the threads: leave the pool, run the plain loop */
        fprintf(stderr, "nhd_oracle_solve_mt: only %d of %d threads\n", started, n_threads);
        abort();
    }
    for (int i = 0; i < n_pods; i++) {
        o_pod top;
        expand_pod(&pods[i], &top);
        nhd_binding* b = &out[i];
        memset(b, 0, sizeof(*b));
        b->node = -1;
        b->n_groups = (uint8_t)top.n_groups;
        if (top.map_type != NHD_MAP_NUMA && top.map_type != NHD_MAP_PCI) { b->status = NHD_BAD_MAP_TYPE; continue; }
        pl.top = &top; pl.now = now[i];
        pthread_barrier_wait(&pl.start);
        pool_do_range(&pl, 0);
        pthread_barrier_wait(&pl.done);
        scan_res sr;
        scan_merge(pl.parts, n_threads, &sr);
        finish_scheduling(nodes, &top, now[i], b, &sr);
        if (b->node >= 0)
            collapse_node(&nodes[b->node], &recs[b->node]);
    }
    pl.quit = 1;
    pthread_barrier_wait(&pl.start);
    for (int t = 1; t < n_threads; t++) pthread_join(th[t], NULL);
    pthread_barrier_destroy(&pl.start); pthread_barrier_destroy(&pl.done);
    free(pl.parts); free(th); free(ws); free(nodes);
    return 0;
}

int nhd_oracle_candidates(const nhd_oracle_params* params, const double* speed_gbps,
                          int n_nodes, const nhd_node_rec* recs,
                          const nhd_pod* pod, double now, uint8_t* cand_out)
{
    P = params; SPEED = speed_gbps;
    o_node* nodes = (o_node*)malloc(sizeof(o_node) * (size_t)(n_nodes > 0 ? n_nodes : 1));
    if (!nodes) return -1;
    for (int n = 0; n < n_nodes; n++) expand_node(&recs[n], &nodes[n]);
    o_pod top;
    expand_pod(pod, &top);
    nhd_binding b;
    attempt_scheduling(nodes, n_nodes, &top, now, &b, cand_out);
    free(nodes);
    return 0;
}
