/*
 * nhd_api.cu — the C-ABI of include/nhd_b200.h on top of the sm_90a kernels.
 *
 * Host side of the drop-in boundary: owns the device mirror of the cluster (tiled node
 * records in HBM), de-duplicates the pod descriptors of a batch into pod types, launches
 * the snapshot predicate kernel and the select+assign sweep, and (when the node set is
 * sharded over several GPUs) merges the per-rank feasibility bitmaps with one NCCL
 * all-reduce.  There is no CPU fallback: every entry point that computes fails with
 * NHD_ERR_CUDA when no device is usable.
 */
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "../../include/nhd_b200.h"
#include "nhd_kernels.cuh"

using namespace nhd;

/* ------------------------------------------------------------------ NCCL, resolved at run time */

typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId_;
typedef int ncclResult_t_;
enum { NCCL_INT8 = 0 };                       /* ncclInt8 / ncclChar (nccl.h, stable since 2.0) */

struct NcclApi {
    void* lib = nullptr;
    ncclResult_t_ (*GetUniqueId)(ncclUniqueId_*) = nullptr;
    ncclResult_t_ (*CommInitRank)(ncclComm_t*, int, ncclUniqueId_, int) = nullptr;
    ncclResult_t_ (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t_ (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t_) = nullptr;
    bool load()
    {
        if (lib) return true;
        /* reuse the copy already mapped into the process (e.g. PyTorch's) before opening the system one */
        lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        if (!lib) lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
        if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_LOCAL);
        if (!lib) return false;
        GetUniqueId = (decltype(GetUniqueId))dlsym(lib, "ncclGetUniqueId");
        CommInitRank = (decltype(CommInitRank))dlsym(lib, "ncclCommInitRank");
        CommDestroy = (decltype(CommDestroy))dlsym(lib, "ncclCommDestroy");
        AllGather = (decltype(AllGather))dlsym(lib, "ncclAllGather");
        GetErrorString = (decltype(GetErrorString))dlsym(lib, "ncclGetErrorString");
        return GetUniqueId && CommInitRank && CommDestroy && AllGather;
    }
};
static NcclApi g_nccl;

static_assert(offsetof(nhd_node_rec, flags) == 2 * 16 + REC_FLAGS_BYTE, "exclude_nodes_kernel's flags byte");
static_assert(sizeof(nhd_release) == 88 && offsetof(nhd_release, nic_pairings) == 56, "nhd_release is 88 bytes");

/* ------------------------------------------------------------------ buffers */

/* An owned device (or pinned host) allocation: grow(bytes) keeps it when it holds that many bytes and otherwise replaces
 * it, contents lost, by one of max(bytes, 256) bytes.  Freed with its owner. */
template <typename T, bool Pinned>
struct Buf {
    T* p = nullptr;
    size_t cap = 0;
    Buf() = default;
    Buf(const Buf&) = delete;
    Buf& operator=(const Buf&) = delete;
    ~Buf() { release(); }
    operator T*() const { return p; }
    void swap(Buf& o) { std::swap(p, o.p); std::swap(cap, o.cap); }
    void release()
    {
        if (p) Pinned ? cudaFreeHost(p) : cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    cudaError_t grow(size_t need)
    {
        if (need <= cap) return cudaSuccess;
        release();
        const size_t want = std::max(need, (size_t)256);
        const cudaError_t e = Pinned ? cudaMallocHost((void**)&p, want) : cudaMalloc((void**)&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
};
template <typename T> using DevBuf = Buf<T, false>;
template <typename T> using PinnedBuf = Buf<T, true>;

/*
 * One solve's pod set and every buffer its kernels write (stage_pods fills and sizes it).  The handle holds two: batch,
 * the staged batch that nhd_solve_staged commits and the explanations and nhd_read_filter read, and scratch, which every
 * query and plan uses, so that those leave the staged batch, its bindings and its filter output alone.
 */
struct Workspace {
    /* the pod set */
    int n_pods = 0, n_types = 0, n_names = 0;
    int pod_cap = 0;                      /* pods the arrays are laid out for: n_pods as staged (a plan's later rounds hold fewer) */
    int seg = 0;                          /* first pod of the solve: a plan with releases solves a round in segments */
    uint64_t names_used = 0;
    double now0 = 0.0;                    /* clock of the first pod (the filter's BUSY row) */
    bool const_clock = true;
    DevBuf<PodType> types;
    DevBuf<uint8_t> pod_arrays;           /* pod_type | now | group masks (when n_names > 0) */
    PinnedBuf<uint8_t> staging;           /* types | pod_arrays */
    std::vector<int32_t> pod_type_host;
    /* the filter's output */
    DevBuf<uint64_t> bitmaps;             /* [n_types + 2 + n_names][words] */
    DevBuf<uint4> dyn;                    /* NodeDyn summaries */
    DevBuf<uint8_t> ftab;                 /* direct-path tables, ftab_bytes(FAST_MAX_TYPES) */
    /* the sweep's */
    DevBuf<int32_t> cursors;              /* [max(n_types, 1)][3] */
    DevBuf<int32_t> busy_list;            /* n_super * SUPER_NODES + 64 */
    DevBuf<int32_t> pend;                 /* n_super * SUPER_NODES */
    DevBuf<unsigned long long> prof;      /* debug counters (nhd_debug_counters reads the batch's) */
    /* the bindings */
    DevBuf<nhd_binding> out;              /* n_pods + 8 (spare records for check builds) */
    PinnedBuf<nhd_binding> h_out;         /* bounce buffer of fetch_bindings */

    size_t now_offset() const { return ((size_t)pod_cap * 4 + 15) & ~(size_t)15; }
    const int32_t* pod_type() const { return reinterpret_cast<const int32_t*>(pod_arrays.p) + seg; }
    const double* now() const { return reinterpret_cast<const double*>(pod_arrays.p + now_offset()) + seg; }
    const uint64_t* pod_groups() const      /* per-pod node-group masks when the pods mix lists, else null */
    {
        return n_names ? reinterpret_cast<const uint64_t*>(pod_arrays.p + now_offset() + (size_t)pod_cap * 8) + seg : nullptr;
    }
    nhd_binding* bindings() const { return out.p + seg; }
};

/* ------------------------------------------------------------------ handle */

struct nhd_handle {
    nhd_params params;
    double cap[NHD_MAX_SPEED_CLASSES];
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    int sm_count = 132;
    int smem_optin = 48 * 1024;
    ncclComm_t comm = nullptr;

    /* cluster mirror */
    int n_nodes = 0, n_super = 0, words = 0, max_numa = 1;
    /* NUMA count of every node the filter could accept (active, not in maintenance; 0 otherwise): the mapping stage's
       tuple limits are judged against the largest of these, and follow updates in both directions */
    std::vector<uint8_t> node_numa;
    int numa_hist[NHD_MAX_NUMA + 1] = {0, 0, 0, 0, 0};
    /* ... as they were at the last nhd_snapshot: nhd_restore puts them back with the records */
    std::vector<uint8_t> snap_node_numa;
    int snap_numa_hist[NHD_MAX_NUMA + 1] = {0, 0, 0, 0, 0};
    int snap_max_numa = 1;
    DevBuf<uint8_t> d_nodes, d_snapshot;
    size_t nodes_bytes = 0;
    bool loaded = false, have_snapshot = false;
    DevBuf<uint16_t> d_class;             /* hardware class of every node of the mirror */
    DevBuf<ClassSlot> d_class_slots;
    DevBuf<ClsFast> d_cls_fast;           /* per hardware class */
    DevBuf<uint32_t> d_sigs;              /* per-NUMA NIC signatures */
    DevBuf<uint8_t> d_mapt;               /* GetNumaGroupIdx table of the direct path */
    uint8_t* d_mapt2 = nullptr;           /* ... with the GPU stage (resolve_kernel); the device's shared copy, not owned */
    DevBuf<uint64_t> d_memo;
    DevBuf<int> d_vresult;
    DevBuf<uint8_t> d_xchg;               /* node-sharded ranks: one slot per rank (summaries + bitmap columns) */

    /* staging for records (AoS) */
    DevBuf<uint8_t> d_stage;
    PinnedBuf<uint8_t> h_stage;
    DevBuf<int32_t> d_idx;

    Workspace batch, scratch;
    bool staged = false, solved = false;
#ifdef NHD_CHECKS
    unsigned long long* d_prof = nullptr;  /* the batch's sweep counters, mapped host: readable after a device fault */
#endif
    long long shard_min_pairs = 1LL << 21;   /* nhd_shard_min_pairs() when the handle was created */

    /* Generation of the device mirror: every call that changes it (or the staged batch) takes a new value.  The
     * explanations need the snapshot to be the batch's starting state and the mirror to hold exactly that batch's
     * commit, i.e. snapshot, stage and solve as three consecutive generations. */
    uint64_t gen = 1, snap_gen = 0, stage_gen = 0, explain_gen = 0;
    bool batch_on_snapshot = false;
    /* explanation scratch: per-node placement lists (CSR), the failed pods, per-pod counts, one pod's node reasons */
    DevBuf<int32_t> d_xnode;              /* node_cnt | node_start | cursor */
    DevBuf<int32_t> d_xpod;               /* node_pods | failed */
    DevBuf<uint32_t> d_xcounts;
    DevBuf<uint8_t> d_xreasons;
    DevBuf<uint32_t> d_xsmall;            /* n_failed, survivors */

    /* Records generation: load and update change it, snapshot remembers it.  A query of the snapshot needs the two
     * equal, so that the nodes' hardware classes (d_class, d_cls_fast, d_sigs: the mirror's) describe the snapshot. */
    uint64_t rec_gen = 1, snap_rec_gen = 0;
    /* a plan's copy of the records, with its excluded nodes flagged there, and their indices */
    DevBuf<uint8_t> d_pnodes;
    DevBuf<int32_t> d_pidx;
    /* a plan's rounds (nhd_plan_batch_rounds): the other half of the scratch pod arrays, both caller-row maps | the round
     * that placed each pod | survivors per CTA, every pod's last attempt, the last round's reason rows, and the word the
     * device leaves the next round's pod count in */
    DevBuf<uint8_t> d_rpods;
    DevBuf<int32_t> d_ridx;
    DevBuf<nhd_binding> d_rout;
    DevBuf<uint32_t> d_rwhy;
    PinnedBuf<int32_t> h_rcount;
    /* a plan's arrivals (nhd_plan_batch_arrivals): the staged pods, apart from the scans' double buffers | the clock of
     * each pod's last attempt */
    DevBuf<uint8_t> d_apods;
    DevBuf<double> d_rclock;
    /* a plan's releases (nhd_plan_batch_releases): the records a segment started from, the releases, and counts |
     * node -> tracked slot | release -> slot | releases by round and node | node starts | the check word */
    DevBuf<uint8_t> d_pseg;
    DevBuf<nhd_release> d_rels;
    DevBuf<int32_t> d_rel;
    /* scenario plans: pod offsets | exclusion offsets | exclusions | edit offsets | edited nodes | lift indices | slot
     * nodes | the failed-mapping word, and one working record per slot followed by the edit records */
    DevBuf<int32_t> d_sidx;
    DevBuf<uint4> d_swork;

    nhd_timing timing;
    std::string err;
};

static int32_t fail(nhd_handle* h, int32_t code, const char* fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (h) h->err = buf;
    return code;
}

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess)                                                                     \
            return fail(h, NHD_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_),   \
                        __FILE__, __LINE__);                                                       \
    } while (0)

/* the sweep's debug counters of w: a check build keeps the batch's in mapped host memory (nhd_create) */
static unsigned long long* counters(nhd_handle* h, Workspace& w)
{
#ifdef NHD_CHECKS
    if (&w == &h->batch) return h->d_prof;
#endif
    return w.prof;
}

/* ------------------------------------------------------------------ validation */

extern "C" int32_t nhd_validate_node(const nhd_node_rec* r)
{
    if (!r) return NHD_ERR_INVALID;
    return validate_node_rec(*r);          /* same routine the upload path runs on the device */
}

extern "C" int32_t nhd_validate_pod(const nhd_pod* p)
{
    if (!p) return NHD_ERR_INVALID;
    if (p->n_groups < 1) return NHD_ERR_INVALID;             /* zero groups crashes the reference (Matcher.py:346) */
    if (p->n_groups > NHD_MAX_GROUPS) return NHD_ERR_UNSUPPORTED;
    int cores = p->n_misc, gpus = 0;
    for (int g = 0; g < p->n_groups; g++) {
        const nhd_pod_group& pg = p->groups[g];
        if (pg.n_gpus > NHD_MAX_GROUP_GPUS) return NHD_ERR_UNSUPPORTED;
        cores += pg.n_proc + pg.n_helpers;
        for (int j = 0; j < pg.n_gpus; j++) cores += pg.gpu_feeders[j];
        gpus += pg.n_gpus;
        if (!(pg.rx_gbps >= 0.0) || !(pg.tx_gbps >= 0.0) || !std::isfinite(pg.rx_gbps) || !std::isfinite(pg.tx_gbps))
            return NHD_ERR_INVALID;
    }
    if (cores > NHD_MAX_POD_CORES || gpus > NHD_MAX_POD_GPUS) return NHD_ERR_UNSUPPORTED;
    return NHD_OK;
}

/* numa^(groups+1) enumeration limits of the mapping stage */
static bool tuple_limits_ok(int K, int G)
{
    long nq = 1, np = 1;
    for (int i = 0; i < G + 1; i++) nq *= K;
    for (int i = 0; i < G; i++) np *= K;
    return nq <= NHD_MAX_TUPLES && np <= 64;
}

static inline uint8_t schedulable_numa(const nhd_node_rec& r)
{
    /* (a record not validated yet may say anything: counts beyond the limit are not counted — the load is rejected) */
    return ((r.flags & NHD_NODE_ACTIVE) && !(r.flags & NHD_NODE_MAINTENANCE) && r.n_numa <= NHD_MAX_NUMA) ? (uint8_t)r.n_numa : (uint8_t)0;
}

static void track_numa(nhd_handle* h, int n, const nhd_node_rec* recs, const int32_t* idx)
{
    for (int i = 0; i < n; i++) {
        const int node = idx ? idx[i] : i;
        const uint8_t k = schedulable_numa(recs[i]);
        h->numa_hist[h->node_numa[node]]--;
        h->numa_hist[k]++;
        h->node_numa[node] = k;
    }
    h->max_numa = 1;
    for (int k = 2; k <= NHD_MAX_NUMA; k++) if (h->numa_hist[k] > 0) h->max_numa = k;
}

/* ------------------------------------------------------------------ lifecycle */

extern "C" void nhd_default_params(nhd_params* p)
{
    if (!p) return;
    memset(p, 0, sizeof(*p));
    p->nic_bw_avail_percent = 0.9;       /* Node.py:18 */
    p->min_busy_secs = 30.0;             /* Node.py:107 */
    p->enable_sharing = 0;               /* Node.py:20 */
    p->world_size = 1;
}

/*
 * Node-sharding threshold: (nodes x distinct pod types) from which the snapshot filter is split over the ranks.
 * Below it every rank filters the whole cluster and no collective runs.  The default was chosen where an earlier GPU's
 * all-gather + unpack of the bitmaps cost more than the shard saves; the whole filter of 65 536 nodes x 16 types takes
 * 0.05 ms on one H100 SXM (400 W power limit), but the exchange cost on H100s has not been measured, so the threshold
 * is carried over unchanged.  Every rank must use the same
 * value (it decides whether the collective is entered): NHD_SHARD_MIN_PAIRS in the environment of all ranks, read
 * when a handle is created; default 2^21.
 */
static long long shard_min_pairs_now()
{
    const char* e = getenv("NHD_SHARD_MIN_PAIRS");
    if (e && *e) {
        char* end = nullptr;
        const long long v = strtoll(e, &end, 10);
        if (end && *end == 0 && v >= 0) return v;
    }
    return 1LL << 21;
}
extern "C" int64_t nhd_shard_min_pairs(void) { return (int64_t)shard_min_pairs_now(); }

extern "C" int32_t nhd_nccl_unique_id(uint8_t out[128])
{
    if (!out) return NHD_ERR_INVALID;
    if (!g_nccl.load()) return NHD_ERR_NCCL;
    ncclUniqueId_ id;
    if (g_nccl.GetUniqueId(&id) != 0) return NHD_ERR_NCCL;
    memcpy(out, id.internal, 128);
    return NHD_OK;
}

/* MAPT2 (mapt2_kernel) is a constant of the CPython set model, 64 KB: one copy per device for the life of the process,
 * shared by every handle on that device and never freed.  Published only after the kernel that fills it has finished. */
static std::mutex g_mapt2_mu;
static uint8_t* g_mapt2[64];
static cudaError_t shared_mapt2(int device, cudaStream_t st, uint8_t** out)
{
    std::lock_guard<std::mutex> lk(g_mapt2_mu);
    if (device < 0 || device >= 64) return cudaErrorInvalidValue;
    if (!g_mapt2[device]) {
        uint8_t* t = nullptr;
        cudaError_t e = cudaMalloc((void**)&t, (size_t)MAPT2_BYTES);
        if (e != cudaSuccess) return e;
        mapt2_kernel<<<(MAPT2_BYTES + 127) / 128, 128, 0, st>>>(t);
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { cudaFree(t); return e; }
        g_mapt2[device] = t;
    }
    *out = g_mapt2[device];
    return cudaSuccess;
}

extern "C" int32_t nhd_destroy(nhd_handle* h)
{
    if (!h) return NHD_OK;
    if (h->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(h->comm);
    cudaSetDevice(h->params.device);
    if (h->stream) cudaStreamSynchronize(h->stream);
#ifdef NHD_CHECKS
    cudaFreeHost(h->d_prof);
#endif
    const cudaStream_t stream = h->stream;
    cudaEvent_t ev[4];
    std::copy(std::begin(h->ev), std::end(h->ev), ev);
    delete h;                                            /* frees every buffer */
    for (auto& e : ev) if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
    return NHD_OK;
}

extern "C" int32_t nhd_create(const nhd_params* p, nhd_handle** out)
{
    if (!p || !out) return NHD_ERR_INVALID;
    *out = nullptr;
    if (p->enable_sharing) return NHD_ERR_UNSUPPORTED;        /* the reference ships with sharing off (Node.py:20) */
    if (p->n_speed_classes < 0 || p->n_speed_classes > NHD_MAX_SPEED_CLASSES) return NHD_ERR_INVALID;
    if (p->world_size < 1 || p->rank < 0 || p->rank >= p->world_size) return NHD_ERR_INVALID;
    nhd_handle* h = new nhd_handle();
    h->params = *p;
    memset(&h->timing, 0, sizeof(h->timing));
    for (int i = 0; i < NHD_MAX_SPEED_CLASSES; i++)
        h->cap[i] = p->speed_gbps[i] * p->nic_bw_avail_percent;   /* n.speed*NIC_BW_AVAIL_PERCENT, Node.py:292 */
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0 || p->device < 0 || p->device >= ndev) {
        delete h;
        return NHD_ERR_CUDA;                                    /* no CPU fallback */
    }
    *out = h;
    h->shard_min_pairs = shard_min_pairs_now();
    CK(cudaSetDevice(p->device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, p->device));
    h->sm_count = prop.multiProcessorCount;
    h->smem_optin = (int)prop.sharedMemPerBlockOptin;
    CK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    for (auto& ev : h->ev) CK(cudaEventCreate(&ev));
    CK(h->d_memo.grow((size_t)MEMO_SLOTS * 16));
    CK(cudaMemsetAsync(h->d_memo, 0, (size_t)MEMO_SLOTS * 16, h->stream));
    CK(h->d_vresult.grow(16));
#ifdef NHD_CHECKS
    CK(cudaHostAlloc((void**)&h->d_prof, 64 * 8, cudaHostAllocMapped));      /* readable after a device fault */
    memset(h->d_prof, 0, 64 * 8);
#else
    CK(h->batch.prof.grow(64 * 8));
    CK(cudaMemsetAsync(h->batch.prof, 0, 64 * 8, h->stream));
#endif
    CK(h->d_class_slots.grow((size_t)CLASS_SLOTS * sizeof(ClassSlot)));
    CK(cudaMemsetAsync(h->d_class_slots, 0, (size_t)CLASS_SLOTS * sizeof(ClassSlot), h->stream));
    CK(h->d_mapt.grow((size_t)((MAPT_BYTES + 15) & ~15)));
    CK(h->d_sigs.grow((size_t)FAST_NSIG * 4));
    CK(cudaMemsetAsync(h->d_sigs, 0, (size_t)FAST_NSIG * 4, h->stream));
    CK(h->d_cls_fast.grow((size_t)CLASS_SLOTS * sizeof(ClsFast)));
    CK(cudaMemsetAsync(h->d_cls_fast, 0, (size_t)CLASS_SLOTS * sizeof(ClsFast), h->stream));
    mapt_kernel<<<(MAPT_BYTES + 127) / 128, 128, 0, h->stream>>>(h->d_mapt);
    CK(cudaGetLastError());
    CK(shared_mapt2(p->device, h->stream, &h->d_mapt2));
    CK(cudaFuncSetAttribute(filter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            FILTER_STAGES * SUPER_BYTES + TYPES_SMEM_MAX * (int)sizeof(PodType)));
    CK(cudaFuncSetAttribute(sweep_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin));
    CK(cudaFuncSetAttribute(sweep_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
    {
        /* one empty launch of the big kernel: its code is loaded (lazy module loading) and resident before the first
         * real batch instead of inside it (a first sweep used to take tens of milliseconds) */
        SweepArgs sa;
        memset(&sa, 0, sizeof(sa));
        sa.prof = counters(h, h->batch);                   /* (profile builds flush their counters) */
        const size_t smem = (size_t)SMEMO_SLOTS * 16 + (size_t)DMEMO_SLOTS * 48 + (size_t)DCACHE_SLOTS * 36 + 16 +
                            (size_t)CLSNIC_SLOTS * 48 + (size_t)SPMEMO_SLOTS * 16 + ((MAPT_BYTES + 15) & ~15) + 4096;
        sweep_kernel<true><<<1, SWEEP_THREADS, smem, h->stream>>>(sa);
        sweep_kernel<false><<<1, SWEEP_THREADS, smem, h->stream>>>(sa);
        CK(cudaGetLastError());
    }
    if (p->world_size > 1) {
        if (!g_nccl.load()) return fail(h, NHD_ERR_NCCL, "libnccl.so.2 not loadable");
        ncclUniqueId_ id;
        memcpy(id.internal, p->nccl_unique_id, 128);
        ncclResult_t_ r = g_nccl.CommInitRank(&h->comm, p->world_size, id, p->rank);
        if (r != 0) return fail(h, NHD_ERR_NCCL, "ncclCommInitRank: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    }
    CK(cudaStreamSynchronize(h->stream));
    return NHD_OK;
}

extern "C" const char* nhd_last_error(const nhd_handle* h) { return h ? h->err.c_str() : "null handle"; }

/* ------------------------------------------------------------------ cluster mirror */

static bool is_pinned_host(const void* p)
{
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeHost;
}

/* hardware classes of the mirror's nodes idx[0..n) (all of [0, n) when idx is null), then the per-class tables */
static int32_t classify(nhd_handle* h, const int32_t* d_idx, int n)
{
    const int threads = 256;
    classify_claim_kernel<<<(n + threads - 1) / threads, threads, 0, h->stream>>>(h->d_nodes, d_idx, n, h->d_class_slots, h->d_class);
    CK(cudaGetLastError());
    classify_verify_kernel<<<(n + threads - 1) / threads, threads, 0, h->stream>>>(h->d_nodes, d_idx, n, h->d_class_slots, h->d_class);
    cls_fast_kernel<<<(CLASS_SLOTS + 255) / 256, 256, 0, h->stream>>>(h->d_class_slots, h->d_cls_fast, h->d_sigs);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(h->stream));
    return NHD_OK;
}

/* host -> device, ingest into the tiled layout, validate on the device, classify.  Records that
 * already sit in pinned memory (nhd_alloc_pinned) are copied straight from the caller's buffer. */
static int32_t upload_records(nhd_handle* h, int n, const nhd_node_rec* recs, const int32_t* idx, int* max_numa,
                              bool track_while_copying = false)
{
    const size_t bytes = (size_t)n * sizeof(nhd_node_rec);
    CK(h->d_stage.grow(bytes));
    const void* src = recs;
    if (!is_pinned_host(recs)) {
        CK(h->h_stage.grow(bytes));
        memcpy(h->h_stage, recs, bytes);
        src = h->h_stage;
    }
    CK(cudaMemcpyAsync(h->d_stage, src, bytes, cudaMemcpyHostToDevice, h->stream));
    const int32_t* d_idx = nullptr;
    if (idx) {
        CK(h->d_idx.grow((size_t)n * 4));
        CK(cudaMemcpyAsync(h->d_idx, idx, (size_t)n * 4, cudaMemcpyHostToDevice, h->stream));
        d_idx = h->d_idx;
    }
    const int threads = 256;
    int vinit[4] = {0x7FFFFFFF, 0, 1, 0};
    CK(cudaMemcpyAsync(h->d_vresult, vinit, 16, cudaMemcpyHostToDevice, h->stream));
    validate_kernel<<<(n + threads - 1) / threads, threads, 0, h->stream>>>((const nhd_node_rec*)h->d_stage.p, n, h->d_vresult);
    CK(cudaGetLastError());
    int vres[4];
    CK(cudaMemcpyAsync(vres, h->d_vresult, 16, cudaMemcpyDeviceToHost, h->stream));
    /* full load: the host's own walk over the records (NUMA bookkeeping) runs while the copy and the validation are in
     * flight; a rejected load leaves the handle unloaded, and the next load starts that bookkeeping afresh */
    if (track_while_copying) track_numa(h, n, recs, idx);
    CK(cudaStreamSynchronize(h->stream));
    if (vres[0] != 0x7FFFFFFF) {
        const int32_t v = nhd_validate_node(&recs[vres[0]]);
        return fail(h, v != NHD_OK ? v : NHD_ERR_INVALID, "node record %d rejected by nhd_validate_node", vres[0]);
    }
    *max_numa = vres[2];
    const int total = n * REC_CHUNKS;
    ingest_kernel<<<(total + threads - 1) / threads, threads, 0, h->stream>>>(
        (const uint4*)h->d_stage.p, d_idx, n, h->d_nodes);
    CK(cudaGetLastError());
    return classify(h, d_idx, n);
}

extern "C" int32_t nhd_load_nodes(nhd_handle* h, int32_t n_nodes, const nhd_node_rec* recs)
{
    if (!h || n_nodes < 0 || (n_nodes > 0 && !recs)) return NHD_ERR_INVALID;
    h->gen++;
    h->rec_gen++;
    CK(cudaSetDevice(h->params.device));
    const int n_super = std::max(1, (n_nodes + SUPER_NODES - 1) / SUPER_NODES);
    const size_t bytes = (size_t)n_super * SUPER_BYTES;
    if (bytes != h->nodes_bytes) {
        h->d_nodes.release(); h->d_snapshot.release(); h->d_class.release();
        h->nodes_bytes = 0;
        CK(h->d_nodes.grow(bytes));
        CK(h->d_snapshot.grow(bytes));
        CK(h->d_class.grow((size_t)n_super * SUPER_NODES * sizeof(uint16_t)));
        h->nodes_bytes = bytes;
    }
    h->n_nodes = n_nodes;
    h->n_super = n_super;
    h->words = n_super * SUPER_NODES / 64;
    CK(cudaMemsetAsync(h->d_nodes, 0, bytes, h->stream));     /* padding nodes: inactive */
    CK(cudaMemsetAsync(h->d_class, 0xFF, (size_t)n_super * SUPER_NODES * sizeof(uint16_t), h->stream));
    h->loaded = true;
    h->have_snapshot = false;
    h->staged = h->solved = false;
    h->max_numa = 1;
    h->node_numa.assign((size_t)n_nodes, 0);
    for (int k = 0; k <= NHD_MAX_NUMA; k++) h->numa_hist[k] = 0;
    h->numa_hist[0] = n_nodes;
    if (n_nodes == 0) { CK(cudaStreamSynchronize(h->stream)); return NHD_OK; }
    int mx = 1;
    const int32_t rc = upload_records(h, n_nodes, recs, nullptr, &mx, true);
    if (rc != NHD_OK) { h->loaded = false; return rc; }
    return NHD_OK;
}

extern "C" int32_t nhd_update_nodes(nhd_handle* h, int32_t n, const int32_t* idx, const nhd_node_rec* recs)
{
    if (!h || n < 0 || (n > 0 && (!idx || !recs))) return NHD_ERR_INVALID;
    if (!h->loaded) return fail(h, NHD_ERR_STATE, "nhd_update_nodes before nhd_load_nodes");
    CK(cudaSetDevice(h->params.device));
    {
        std::vector<uint8_t> seen((size_t)h->n_nodes, 0);            /* the device applies the records in parallel: one per node */
        for (int i = 0; i < n; i++) {
            if (idx[i] < 0 || idx[i] >= h->n_nodes) return fail(h, NHD_ERR_INVALID, "node index %d out of range", idx[i]);
            if (seen[idx[i]]) return fail(h, NHD_ERR_INVALID, "node index %d appears twice in one update", idx[i]);
            seen[idx[i]] = 1;
            int32_t v = nhd_validate_node(&recs[i]);      /* before anything is written: an update must not half-apply */
            if (v != NHD_OK) return fail(h, v, "update %d: record rejected", i);
        }
    }
    if (n == 0) return NHD_OK;
    h->gen++;
    h->rec_gen++;
    int mx = 1;
    const int32_t rc = upload_records(h, n, recs, idx, &mx);
    if (rc == NHD_OK) track_numa(h, n, recs, idx);
    return rc;
}

extern "C" int32_t nhd_read_nodes(nhd_handle* h, int32_t first, int32_t n, nhd_node_rec* out)
{
    if (!h || first < 0 || n < 0 || (n > 0 && !out)) return NHD_ERR_INVALID;
    if (!h->loaded || (long long)first + (long long)n > (long long)h->n_nodes) return fail(h, NHD_ERR_STATE, "range outside the loaded cluster");
    if (n == 0) return NHD_OK;
    CK(cudaSetDevice(h->params.device));
    const size_t bytes = (size_t)n * sizeof(nhd_node_rec);
    CK(h->d_stage.grow(bytes));
    CK(h->h_stage.grow(bytes));
    const int threads = 256, total = n * REC_CHUNKS;
    export_kernel<<<(total + threads - 1) / threads, threads, 0, h->stream>>>(h->d_nodes, first, n, (uint4*)h->d_stage.p);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(h->h_stage, h->d_stage, bytes, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    memcpy(out, h->h_stage, bytes);
    return NHD_OK;
}

extern "C" int32_t nhd_snapshot(nhd_handle* h)
{
    if (!h) return NHD_ERR_STATE;
    if (!h->loaded) return fail(h, NHD_ERR_STATE, "nhd_snapshot before nhd_load_nodes");
    CK(cudaSetDevice(h->params.device));
    h->gen++;
    CK(cudaMemcpyAsync(h->d_snapshot, h->d_nodes, h->nodes_bytes, cudaMemcpyDeviceToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    h->have_snapshot = true;
    h->snap_gen = h->gen;
    h->snap_rec_gen = h->rec_gen;
    h->snap_node_numa = h->node_numa;
    memcpy(h->snap_numa_hist, h->numa_hist, sizeof(h->numa_hist));
    h->snap_max_numa = h->max_numa;
    return NHD_OK;
}

/* The snapshot's records back into the mirror, with the tuple-limit bookkeeping they had.  After an nhd_update_nodes
 * the mirror's hardware classes describe the updated records, so every node is classified again. */
extern "C" int32_t nhd_restore(nhd_handle* h)
{
    if (!h) return NHD_ERR_STATE;
    if (!h->loaded || !h->have_snapshot)
        return fail(h, NHD_ERR_STATE, "nhd_restore needs an nhd_snapshot since the last nhd_load_nodes");
    h->gen++;
    CK(cudaSetDevice(h->params.device));
    CK(cudaMemcpyAsync(h->d_nodes, h->d_snapshot, h->nodes_bytes, cudaMemcpyDeviceToDevice, h->stream));
    h->node_numa = h->snap_node_numa;
    memcpy(h->numa_hist, h->snap_numa_hist, sizeof(h->numa_hist));
    h->max_numa = h->snap_max_numa;
    if (h->rec_gen != h->snap_rec_gen && h->n_nodes > 0) return classify(h, nullptr, h->n_nodes);
    return NHD_OK;
}

/* ------------------------------------------------------------------ batch: stage / solve / fetch */

extern "C" int32_t nhd_sync(nhd_handle* h);

struct PodKey {
    nhd_pod p;
    bool operator==(const PodKey& o) const { return memcmp(&p, &o.p, sizeof(nhd_pod)) == 0; }
};
struct PodKeyHash {
    size_t operator()(const PodKey& k) const
    {
        const uint64_t* w = reinterpret_cast<const uint64_t*>(&k.p);
        uint64_t h = 0x9E3779B97F4A7C15ULL;
        for (size_t i = 0; i < sizeof(nhd_pod) / 8; i++) { h ^= w[i]; h *= 0xff51afd7ed558ccdULL; h ^= h >> 29; }
        return (size_t)h;
    }
};

/* normalise a descriptor so that equal requests compare equal bytewise */
static nhd_pod canonical_pod(const nhd_pod& in)
{
    nhd_pod p;
    memset(&p, 0, sizeof(p));
    p.n_groups = in.n_groups; p.map_type = in.map_type; p.n_misc = in.n_misc;
    p.flags = in.flags & NHD_POD_MISC_SMT;
    p.hugepages_gb = in.hugepages_gb; p.group_mask = in.group_mask;
    for (int g = 0; g < in.n_groups && g < NHD_MAX_GROUPS; g++) {
        nhd_pod_group& o = p.groups[g];
        const nhd_pod_group& i = in.groups[g];
        o.n_gpus = i.n_gpus; o.n_proc = i.n_proc; o.n_helpers = i.n_helpers;
        o.flags = i.flags & (NHD_GRP_PROC_SMT | NHD_GRP_HELPER_SMT | NHD_GRP_HAS_NIC_CORES);
        for (int j = 0; j < i.n_gpus && j < NHD_MAX_GROUP_GPUS; j++) o.gpu_feeders[j] = i.gpu_feeders[j];
        o.rx_gbps = i.rx_gbps + 0.0; o.tx_gbps = i.tx_gbps + 0.0;     /* -0.0 -> +0.0 */
    }
    return p;
}

/* node-group gate (NHDScheduler.py:235-247): one distinct pod group list -> folded into the pod types; several ->
 * types are group-agnostic and the per-name node bitmaps apply the gate.  Returns whether the pods mix lists. */
static bool group_lists(int n_pods, const nhd_pod* pods, uint64_t* names_used)
{
    bool multi_group = false;
    uint64_t used = 0;
    for (int i = 0; i < n_pods; i++) {
        used |= pods[i].group_mask;
        if (pods[i].group_mask != pods[0].group_mask) multi_group = true;
    }
    *names_used = used;
    return multi_group;
}

/* The staging checks of one pod, in order: the descriptor (nhd_validate_pod), a finite clock, the tuple limits against
 * max_numa.  The refusal names the pod as index i; h may be null (the code alone). */
static int32_t check_pod(nhd_handle* h, int i, const nhd_pod& p, double now, int max_numa)
{
    const int32_t v = nhd_validate_pod(&p);
    if (v != NHD_OK) return fail(h, v, "pod %d: descriptor rejected by nhd_validate_pod", i);
    if (!std::isfinite(now)) return fail(h, NHD_ERR_INVALID, "pod %d: non-finite clock", i);
    if (!tuple_limits_ok(max_numa, p.n_groups))
        return fail(h, NHD_ERR_UNSUPPORTED, "pod %d: %d groups on %d-NUMA nodes exceeds the tuple limits", i,
                    (int)p.n_groups, max_numa);
    return NHD_OK;
}

/* Validate the pods and de-duplicate them into pod types (distinct descriptors: the reference re-derives everything
 * per pod): types[] and pod_type[i].  Refusals name the pod; the tuple limits are judged against max_numa.  Touches
 * nothing of the handle but its error text. */
static int32_t make_pod_types(nhd_handle* h, int n_pods, const nhd_pod* pods, const double* now, bool multi_group,
                              int max_numa, std::vector<PodType>& types, std::vector<int32_t>& pod_type)
{
    std::unordered_map<PodKey, int32_t, PodKeyHash> index;
    index.reserve(64);
    types.clear();
    pod_type.resize(n_pods);
    /* pending sets repeat a few descriptors thousands of times: a descriptor seen before (byte for byte) skips
     * validation, normalisation and the map */
    struct RawSlot { uint64_t hash; int32_t type; nhd_pod raw; };
    static thread_local std::vector<RawSlot> raw_cache;
    raw_cache.assign(256, RawSlot{0, -1, {}});
    for (int i = 0; i < n_pods; i++) {
        uint64_t rh = 0x9E3779B97F4A7C15ULL;
        {
            const uint64_t* w = reinterpret_cast<const uint64_t*>(&pods[i]);
            for (size_t q = 0; q < sizeof(nhd_pod) / 8; q++) { rh ^= w[q]; rh *= 0xff51afd7ed558ccdULL; rh ^= rh >> 29; }
        }
        RawSlot& rs = raw_cache[rh & 255];
        if (rs.type >= 0 && rs.hash == rh && memcmp(&rs.raw, &pods[i], sizeof(nhd_pod)) == 0) {
            if (!std::isfinite(now[i])) return fail(h, NHD_ERR_INVALID, "pod %d: non-finite clock", i);
            pod_type[i] = rs.type;
            continue;
        }
        const int32_t v = check_pod(h, i, pods[i], now[i], max_numa);
        if (v != NHD_OK) return v;
        PodKey k{canonical_pod(pods[i])};
        if (multi_group) k.p.group_mask = ~0ULL;
        auto it = index.find(k);
        if (it == index.end()) {
            PodType t;
            memset(&t, 0, sizeof(t));
            make_pod_type(k.p, t);
            it = index.emplace(k, (int32_t)types.size()).first;
            types.push_back(t);
        }
        pod_type[i] = it->second;
        rs.hash = rh; rs.type = it->second; rs.raw = pods[i];
    }
    return NHD_OK;
}

/*
 * Validate a pod set, de-duplicate it into pod types (tuple limits judged against max_numa) and copy it into w: the
 * types, then pod_type | now | group masks, through w's pinned staging.  Every buffer of w is sized here, from the
 * pod set and n_super, so that no allocation falls inside the solve that follows.
 */
static int32_t stage_pods(nhd_handle* h, Workspace& w, int n, const nhd_pod* pods, const double* now, int max_numa)
{
    uint64_t names_used = 0;
    const bool multi_group = group_lists(n, pods, &names_used);
    std::vector<PodType> types;
    const int32_t rc = make_pod_types(h, n, pods, now, multi_group, max_numa, types, w.pod_type_host);
    if (rc != NHD_OK) return rc;
    CK(cudaSetDevice(h->params.device));
    const int T = (int)types.size();
    w.n_pods = w.pod_cap = n;
    w.seg = 0;
    w.n_types = T;
    w.n_names = multi_group ? __builtin_popcountll(names_used) : 0;
    w.names_used = multi_group ? names_used : 0;
    w.now0 = n ? now[0] : 0.0;
    w.const_clock = true;
    for (int i = 1; i < n; i++) if (now[i] != now[0]) { w.const_clock = false; break; }

    const size_t types_bytes = (size_t)T * sizeof(PodType), off_now = w.now_offset(), off_gm = off_now + (size_t)n * 8;
    const size_t pods_bytes = off_gm + (w.n_names ? (size_t)n * 8 : 0), n_slots = (size_t)h->n_super * SUPER_NODES;
    CK(w.staging.grow(types_bytes + pods_bytes));
    CK(w.types.grow(types_bytes));
    CK(w.pod_arrays.grow(pods_bytes));
    CK(w.bitmaps.grow((size_t)(T + 2 + w.n_names) * h->words * 8));
    CK(w.dyn.grow(n_slots * sizeof(NodeDyn)));
    CK(w.ftab.grow(ftab_bytes(FAST_MAX_TYPES)));
    CK(w.cursors.grow((size_t)std::max(T, 1) * 3 * 4));
    CK(w.busy_list.grow((n_slots + 64) * 4));
    CK(w.pend.grow(n_slots * 4));
    CK(w.prof.grow(64 * 8));
    CK(w.out.grow(((size_t)n + 8) * sizeof(nhd_binding)));
    if (n == 0) return NHD_OK;
    uint8_t* hp = w.staging + types_bytes;
    memcpy(w.staging, types.data(), types_bytes);
    memcpy(hp, w.pod_type_host.data(), (size_t)n * 4);
    memcpy(hp + off_now, now, (size_t)n * 8);
    if (w.n_names)
        for (int i = 0; i < n; i++) memcpy(hp + off_gm + (size_t)i * 8, &pods[i].group_mask, 8);
    CK(cudaMemcpyAsync(w.types, w.staging, types_bytes, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(w.pod_arrays, hp, pods_bytes, cudaMemcpyHostToDevice, h->stream));
    return NHD_OK;
}

extern "C" int32_t nhd_stage_batch(nhd_handle* h, int32_t n_pods, const nhd_pod* pods, const double* now)
{
    if (!h || n_pods < 0 || (n_pods > 0 && (!pods || !now))) return NHD_ERR_INVALID;
    if (!h->loaded) return fail(h, NHD_ERR_STATE, "nhd_stage_batch before nhd_load_nodes");
    const bool on_snapshot = h->gen == h->snap_gen;
    h->gen++;
    h->staged = h->solved = false;
    const int32_t rc = stage_pods(h, h->batch, n_pods, pods, now, h->max_numa);
    if (rc != NHD_OK) return rc;
    h->staged = true;
    h->batch_on_snapshot = on_snapshot;
    h->stage_gen = h->gen;
    return NHD_OK;
}

static int32_t solve_staged(nhd_handle* h, bool filter_only);
extern "C" int32_t nhd_solve_staged(nhd_handle* h) { return solve_staged(h, false); }
extern "C" int32_t nhd_run_filter_only(nhd_handle* h)
{
    int32_t r = solve_staged(h, true);
    if (r != NHD_OK) return r;
    return nhd_sync(h);
}

/*
 * The launches of a solve of w's pod set on the records nodes: direct-path tables, filter, sweep, resolve, core ids.
 * batch = the handle's staged batch on the mirror: its timing events and the node-sharded filter + exchange when
 * world_size > 1.  Without it (a plan, or a query's filter) neither: every rank filters the whole cluster.  commit =
 * commit_kernel folds the bindings into nodes (the mirror for the batch, a plan's own copy between its rounds);
 * without it the records are only read.  filter_only stops after the filter.
 */
static int32_t launch_solve(nhd_handle* h, Workspace& w, const uint8_t* nodes, bool batch, bool commit, bool filter_only)
{
    const int T = w.n_types, W = h->words;
    int launches = 0;

    /* 1. snapshot predicate kernel over this rank's node shard.  With several ranks every rank filters the nodes
     * of S consecutive super-tiles into its slot of an exchange buffer (their NodeDyn summaries, then their
     * columns of every bitmap row); one all-gather hands every rank all slots, and a small kernel lays them out
     * as the arrays the (replicated) sweep reads.  Clusters too small for that to pay (nhd_shard_min_pairs) are
     * filtered whole by every rank, without any exchange. */
    const int ws = h->params.world_size, rk = h->params.rank;
    const int rows = T + 2 + w.n_names;
    const size_t bm_bytes = (size_t)rows * W * 8;
    const bool sharded = batch && ws > 1 && w.n_pods > 0 && (long long)h->n_nodes * T >= h->shard_min_pairs;
    const int S = sharded ? (h->n_super + ws - 1) / ws : h->n_super;
    const int super_lo = sharded ? std::min(rk * S, h->n_super) : 0;
    const int super_hi = sharded ? std::min(super_lo + S, h->n_super) : h->n_super;
    const size_t slot_bytes = (size_t)S * 32 * (SUPER_NODES + rows);
    if (sharded) CK(h->d_xchg.grow(slot_bytes * ws));
    if (batch) CK(cudaEventRecord(h->ev[0], h->stream));
    const bool have_ftab = T > 0 && T <= FAST_MAX_TYPES;
    if (w.n_pods > 0 && have_ftab) {
        /* 0. the direct-path tables of this batch's pod types (filter and sweep both read them) */
        TablesArgs ta;
        ta.types = w.types; ta.n_types = T; ta.sigs = h->d_sigs; ta.out = w.ftab;
        memcpy(ta.cap, h->cap, sizeof(ta.cap));
        fast_tables_kernel<<<dim3(T, FAST_NSIG * 16 / 256), 256, 0, h->stream>>>(ta);
        CK(cudaGetLastError());
        launches++;
    }
    if (w.n_pods > 0 && super_hi > super_lo) {
        FilterArgs fa;
        fa.ftab = have_ftab ? w.ftab.p : nullptr; fa.mapt = h->d_mapt; fa.cls = h->d_cls_fast;
        fa.nodes = nodes; fa.types = w.types; fa.n_types = T; fa.n_nodes = h->n_nodes;
        fa.super_lo = super_lo; fa.super_hi = super_hi;
        if (sharded) {
            uint8_t* slot = h->d_xchg + slot_bytes * rk;
            fa.dyn = reinterpret_cast<uint4*>(slot);
            fa.bitmaps = reinterpret_cast<uint64_t*>(slot + (size_t)S * SUPER_NODES * 32);
            fa.words = S * 4; fa.word_base = super_lo * 4;
        } else {
            fa.dyn = w.dyn; fa.bitmaps = w.bitmaps; fa.words = W; fa.word_base = 0;
        }
        fa.class_id = h->d_class; fa.names_used = w.names_used;
        fa.now0 = w.now0; fa.min_busy = h->params.min_busy_secs;
        memcpy(fa.cap, h->cap, sizeof(fa.cap));
        /* few super-tiles (small cluster, or a rank's shard): deal the pod types over several CTAs per super-tile */
        const int n_sh = super_hi - super_lo;
        fa.type_split = std::max(1, std::min(T, (h->sm_count * 2) / n_sh));
        const int grid = std::min(n_sh, h->sm_count * 2) * fa.type_split;
        const size_t smem = FILTER_STAGES * SUPER_BYTES + (T <= TYPES_SMEM_MAX ? (size_t)T * sizeof(PodType) : 0);
        filter_kernel<<<grid, FILTER_THREADS, smem, h->stream>>>(fa);
        CK(cudaGetLastError());
        launches++;
    }
    if (batch) CK(cudaEventRecord(h->ev[1], h->stream));

    /* 2. one collective per batch: every rank contributes its slot */
    if (sharded) {
        ncclResult_t_ r = g_nccl.AllGather(h->d_xchg + slot_bytes * rk, h->d_xchg, slot_bytes, NCCL_INT8, h->comm, h->stream);
        if (r != 0) return fail(h, NHD_ERR_NCCL, "ncclAllGather: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
        const size_t n16 = slot_bytes / 16 * ws;
        uint4* const dyn = w.dyn;
        uint64_t* const bitmaps = w.bitmaps;
        unpack_slots_kernel<<<(unsigned)((n16 + 255) / 256), 256, 0, h->stream>>>(reinterpret_cast<const uint4*>(h->d_xchg.p), ws, S, h->n_super,
                                                                              rows, W, h->n_nodes, h->d_class, dyn, bitmaps);
        CK(cudaGetLastError());
        launches += 2;
    }
    if (batch) CK(cudaEventRecord(h->ev[2], h->stream));

    /* 3. sequential select + assign sweep (replicated on every rank) */
    if (w.n_pods > 0 && !filter_only) {
        /* (the sweep's and the finishing kernels' record pointer is writable for commit_kernel) */
        uint8_t* const records = const_cast<uint8_t*>(nodes);
        SweepArgs sa;
        sa.nodes = records; sa.types = w.types; sa.pod_type = w.pod_type(); sa.now = w.now(); sa.out = w.bindings();
        sa.n_pods = w.n_pods; sa.n_types = T; sa.n_nodes = h->n_nodes; sa.words = W;
        sa.n_names = w.n_names; sa.names_used = w.names_used; sa.pod_groups = w.pod_groups();
        /* reserved_ (test knobs; every setting gives the same bindings): low byte 0 = default, 1 = the general one-warp
         * sweep only (no standing decisions), 2 = standing decisions but never the two pod classes side by side;
         * bits 8.. = debug switches of sweep_kernel */
        sa.dual = (w.const_clock && (h->params.reserved_ & 0xFF) != 1) ? 1 : 0;
        sa.sweep_flags = ((h->params.reserved_ & 0xFF) == 2 ? 1 : 0) | ((h->params.reserved_ >> 8) << 8);
        sa.bitmaps = w.bitmaps; sa.dyn = w.dyn; sa.cursors = w.cursors; sa.busy_list = w.busy_list;
        /* the mapping memo is a pure cache of choose_mapping (its key holds every input: K, G and the three stage
         * masks), so every workspace shares the handle's */
        sa.memo = h->d_memo; sa.prof = counters(h, w); sa.pend_pod = w.pend;
        sa.mapt = h->d_mapt; sa.mapt2 = h->d_mapt2; sa.sigs = h->d_sigs; sa.cls_fast = h->d_cls_fast;
        sa.ftab = (T > 0 && T <= FAST_MAX_TYPES) ? w.ftab.p : nullptr;
        sa.min_busy = h->params.min_busy_secs;
        memcpy(sa.cap, h->cap, sizeof(sa.cap));
        /* shared memory: memo front | pod types | cursors | (bitmaps when they fit) */
        size_t smem = (size_t)SMEMO_SLOTS * 16 + (size_t)DMEMO_SLOTS * 48 + (size_t)DCACHE_SLOTS * 36 + 16 +
                      (size_t)CLSNIC_SLOTS * 48 + (size_t)SPMEMO_SLOTS * 16;
        if (T <= SWEEP_TYPES_SMEM_MAX) smem += (((size_t)T * sizeof(PodType) + 15) & ~(size_t)15) + (size_t)T * 256;
        smem += (((size_t)T * 3 * 4 + 15) & ~(size_t)15) + (size_t)W * 8;
        if (T <= FAST_MAX_TYPES)                /* standing decisions + their tables */
            smem += ftab_small_bytes(T) + (size_t)T * FAST_NSIG_SMEM * 128 + ((MAPT_BYTES + 15) & ~15) +
                    (((size_t)(T + 2) * 4 + 15) & ~(size_t)15);
        const size_t with_bitmaps = smem + bm_bytes;
        /* a second CTA takes the GPU pods when the two pod classes cannot meet (decided on the device, see sweep_kernel) */
        const int sweep_ctas = sa.dual ? 2 : 1;
        if (with_bitmaps <= (size_t)h->smem_optin) {
            sweep_kernel<true><<<sweep_ctas, SWEEP_THREADS, with_bitmaps, h->stream>>>(sa);
        } else {
            sweep_kernel<false><<<sweep_ctas, SWEEP_THREADS, smem, h->stream>>>(sa);
        }
        CK(cudaGetLastError());
        FinishArgs fin;
        fin.nodes = records; fin.types = w.types; fin.pod_type = w.pod_type(); fin.out = w.bindings();
        fin.dyn = w.dyn; fin.n_pods = w.n_pods;
        const int fthreads = 128, fgrid = (w.n_pods + fthreads - 1) / fthreads;
        resolve_kernel<<<(w.n_pods + 63) / 64, 64, 0, h->stream>>>(sa);
        CK(cudaGetLastError());
        assign_cores_kernel<<<fgrid, fthreads, 0, h->stream>>>(fin);
        CK(cudaGetLastError());
        launches += 3;
        if (commit) {
            commit_kernel<<<fgrid, fthreads, 0, h->stream>>>(fin);
            CK(cudaGetLastError());
            launches++;
        }
    }
    if (batch) {
        CK(cudaEventRecord(h->ev[3], h->stream));
        h->timing.n_launches = launches;
        h->timing.n_types = T;
    }
    return NHD_OK;
}

static int32_t solve_staged(nhd_handle* h, bool filter_only)
{
    if (!h) return NHD_ERR_INVALID;
    if (!h->staged) return fail(h, NHD_ERR_STATE, "nhd_solve_staged without a staged batch");
    const bool explainable = !filter_only && h->batch_on_snapshot && h->gen == h->stage_gen;
    h->gen++;
    h->explain_gen = explainable ? h->gen : 0;
    CK(cudaSetDevice(h->params.device));
    const int32_t rc = launch_solve(h, h->batch, h->d_nodes, true, !filter_only, filter_only);
    if (rc != NHD_OK) return rc;
    h->solved = true;
    return NHD_OK;
}

/* device -> host: the first n bindings of w (or of from, when given), through w's bounce buffer unless out is pinned;
 * waits for the device */
static int32_t fetch_bindings(nhd_handle* h, Workspace& w, int n, nhd_binding* out, const nhd_binding* from = nullptr)
{
    const size_t bytes = (size_t)n * sizeof(nhd_binding);
    const bool direct = bytes == 0 || is_pinned_host(out);
    if (!direct) CK(w.h_out.grow(bytes));
    if (bytes) CK(cudaMemcpyAsync(direct ? (void*)out : (void*)w.h_out.p, from ? from : w.out.p, bytes, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (!direct) memcpy(out, w.h_out, bytes);
    return NHD_OK;
}

/* the batch's stage times, once its last event has completed */
static void read_timing(nhd_handle* h)
{
    cudaEventElapsedTime(&h->timing.filter_ms, h->ev[0], h->ev[1]);
    cudaEventElapsedTime(&h->timing.exchange_ms, h->ev[1], h->ev[2]);
    cudaEventElapsedTime(&h->timing.sweep_ms, h->ev[2], h->ev[3]);
    cudaEventElapsedTime(&h->timing.total_ms, h->ev[0], h->ev[3]);
}

extern "C" int32_t nhd_fetch_bindings(nhd_handle* h, nhd_binding* out)
{
    if (!h) return NHD_ERR_INVALID;
    if (!h->solved) return fail(h, NHD_ERR_STATE, "nhd_fetch_bindings without a solved batch");
    CK(cudaSetDevice(h->params.device));
    if (h->batch.n_pods > 0 && !out) return NHD_ERR_INVALID;
    const int32_t rc = fetch_bindings(h, h->batch, h->batch.n_pods, out);
    if (rc != NHD_OK) return rc;
    read_timing(h);
    return NHD_OK;
}

extern "C" int32_t nhd_sync(nhd_handle* h)
{
    if (!h) return NHD_ERR_INVALID;
    CK(cudaSetDevice(h->params.device));
    CK(cudaStreamSynchronize(h->stream));
    if (h->solved) read_timing(h);
    return NHD_OK;
}

extern "C" int32_t nhd_solve_batch(nhd_handle* h, int32_t n_pods, const nhd_pod* pods, const double* now, nhd_binding* out)
{
    int32_t r = nhd_stage_batch(h, n_pods, pods, now);
    if (r != NHD_OK) return r;
    r = nhd_solve_staged(h);
    if (r != NHD_OK) return r;
    return nhd_fetch_bindings(h, out);
}

extern "C" int32_t nhd_last_timing(const nhd_handle* h, nhd_timing* out)
{
    if (!h || !out) return NHD_ERR_INVALID;
    *out = h->timing;
    return NHD_OK;
}

extern "C" int32_t nhd_read_filter(nhd_handle* h, int32_t* n_types, int32_t* words_per_type, uint64_t* words,
                                   int64_t capacity_words, int32_t* pod_type, int32_t n_pods)
{
    if (!h || !h->solved) return NHD_ERR_STATE;
    CK(cudaSetDevice(h->params.device));
    const Workspace& w = h->batch;
    if (n_types) *n_types = w.n_types;
    if (words_per_type) *words_per_type = h->words;
    const int64_t need = (int64_t)(w.n_types + 2) * h->words;    /* group-name bitmaps are not exported */
    if (words) {
        if (capacity_words < need) return NHD_ERR_INVALID;
        CK(cudaMemcpyAsync(words, w.bitmaps, (size_t)need * 8, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
    }
    if (pod_type) {
        if (n_pods < w.n_pods) return NHD_ERR_INVALID;
        memcpy(pod_type, w.pod_type_host.data(), (size_t)w.n_pods * 4);
    }
    return NHD_OK;
}

/* ------------------------------------------------------------------ explanations */

static int32_t explain_ready(nhd_handle* h)
{
    if (!h->solved || h->explain_gen == 0 || h->gen != h->explain_gen)
        return fail(h, NHD_ERR_STATE, "explanations need nhd_snapshot -> nhd_stage_batch -> solve, with nothing changing "
                                      "the device mirror in between or since");
    return NHD_OK;
}

/* The pods of w's solve bound to each node, in pod order (CSR over w.out), and the list of NO_CANDIDATE pods.
 * Returns the number of NO_CANDIDATE pods in *n_failed. */
static int32_t explain_prepare(nhd_handle* h, const Workspace& w, int* n_failed)
{
    const int N = h->n_nodes, P = w.n_pods;
    const nhd_binding* out = w.bindings();
    CK(h->d_xnode.grow(((size_t)3 * N + 2) * 4));
    CK(h->d_xpod.grow(((size_t)2 * P + 1) * 4));
    CK(h->d_xsmall.grow(16));
    int32_t* node_cnt = h->d_xnode;
    int32_t* node_start = h->d_xnode + N;            /* N + 1 entries */
    int32_t* cursor = h->d_xnode + 2 * N + 1;
    int32_t* node_pods = h->d_xpod;
    int32_t* failed = h->d_xpod + P;
    CK(cudaMemsetAsync(node_cnt, 0, (size_t)N * 4, h->stream));
    CK(cudaMemsetAsync(h->d_xsmall, 0, 16, h->stream));
    const int threads = 256;
    if (P > 0) {
        explain_count_kernel<<<(P + threads - 1) / threads, threads, 0, h->stream>>>(out, P, node_cnt, failed,
                                                                                     (int32_t*)h->d_xsmall.p);
        CK(cudaGetLastError());
    }
    explain_scan_kernel<<<1, EXPLAIN_SCAN_THREADS, 0, h->stream>>>(node_cnt, N, node_start, cursor);
    CK(cudaGetLastError());
    if (P > 0) {
        explain_fill_kernel<<<(P + threads - 1) / threads, threads, 0, h->stream>>>(out, P, cursor, node_pods);
        CK(cudaGetLastError());
    }
    if (N > 0) {
        explain_sort_kernel<<<(N + threads - 1) / threads, threads, 0, h->stream>>>(node_start, N, node_pods);
        CK(cudaGetLastError());
    }
    int32_t nf = 0;
    CK(cudaMemcpyAsync(&nf, h->d_xsmall, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    *n_failed = nf;
    return NHD_OK;
}

/* one (failed pod x node) pass over w's solve, which started from the records nodes; counts and/or reasons may be null;
 * d_now (device, per pod) replaces the staged clocks when given */
static int32_t explain_launch(nhd_handle* h, const Workspace& w, const uint8_t* nodes, int n_failed, uint32_t* d_counts,
                              uint8_t* d_reasons, const double* d_now = nullptr)
{
    const int N = h->n_nodes, P = w.n_pods;
    if (n_failed == 0 || N == 0) return NHD_OK;
    ExplainArgs xa;
    xa.snapshot = nodes; xa.types = w.types; xa.pod_type = w.pod_type(); xa.now = d_now ? d_now : w.now(); xa.out = w.bindings();
    xa.pod_groups = w.pod_groups();
    xa.node_start = h->d_xnode + N; xa.node_pods = h->d_xpod; xa.failed = h->d_xpod + P;
    xa.n_failed = (const int32_t*)h->d_xsmall.p;
    xa.n_nodes = N; xa.min_busy = h->params.min_busy_secs;
    memcpy(xa.cap, h->cap, sizeof(xa.cap));
    xa.counts = d_counts; xa.reasons = d_reasons; xa.survivors = h->d_xsmall + 1;
    const dim3 grid((unsigned)((N + EXPLAIN_THREADS - 1) / EXPLAIN_THREADS), (unsigned)std::min(n_failed, 65535));
    explain_kernel<<<grid, EXPLAIN_THREADS, 0, h->stream>>>(xa);
    CK(cudaGetLastError());
    return NHD_OK;
}

/* every NO_CANDIDATE pod's nodes must all be dropped by some stage: a node passing them all means the state was
 * not rebuilt as the pod saw it */
static int32_t explain_survivors(nhd_handle* h, const char* what)
{
    uint32_t surv = 0;
    CK(cudaMemcpyAsync(&surv, h->d_xsmall + 1, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (surv) return fail(h, NHD_ERR_STATE, "%s: %u (pod, node) pairs of NO_CANDIDATE pods pass every stage", what, surv);
    return NHD_OK;
}

/* per-reason node counts of every NO_CANDIDATE pod of w's solve from the records nodes into d_xcounts (n_pods > 0 rows
 * of NHD_WHY_COUNT, zero for the other pods) */
static int32_t explain_rows(nhd_handle* h, const Workspace& w, const uint8_t* nodes)
{
    const size_t bytes = (size_t)w.n_pods * NHD_WHY_COUNT * 4;
    int nf = 0;
    int32_t rc;
    if ((rc = explain_prepare(h, w, &nf)) != NHD_OK) return rc;
    CK(h->d_xcounts.grow(bytes));
    CK(cudaMemsetAsync(h->d_xcounts, 0, bytes, h->stream));
    return explain_launch(h, w, nodes, nf, h->d_xcounts, nullptr);
}

/* ... into the host array counts (n_pods * NHD_WHY_COUNT) */
static int32_t explain_counts(nhd_handle* h, const Workspace& w, const uint8_t* nodes, uint32_t* counts, const char* what)
{
    const size_t bytes = (size_t)w.n_pods * NHD_WHY_COUNT * 4;
    if (bytes == 0) return NHD_OK;
    const int32_t rc = explain_rows(h, w, nodes);
    if (rc != NHD_OK) return rc;
    CK(cudaMemcpyAsync(counts, h->d_xcounts, bytes, cudaMemcpyDeviceToHost, h->stream));
    return explain_survivors(h, what);
}

extern "C" int32_t nhd_explain_batch(nhd_handle* h, uint32_t* counts)
{
    if (!h || (h->batch.n_pods > 0 && !counts)) return NHD_ERR_INVALID;
    int32_t rc = explain_ready(h);
    if (rc != NHD_OK) return rc;
    CK(cudaSetDevice(h->params.device));
    return explain_counts(h, h->batch, h->d_snapshot, counts, "nhd_explain_batch");
}

extern "C" int32_t nhd_explain_pod(nhd_handle* h, int32_t pod, uint8_t* node_reason)
{
    if (!h || (h->n_nodes > 0 && !node_reason)) return NHD_ERR_INVALID;
    int32_t rc = explain_ready(h);
    if (rc != NHD_OK) return rc;
    const Workspace& w = h->batch;
    if (pod < 0 || pod >= w.n_pods) return fail(h, NHD_ERR_INVALID, "pod %d outside the batch of %d", pod, w.n_pods);
    CK(cudaSetDevice(h->params.device));
    int32_t status = 0;
    CK(cudaMemcpyAsync(&status, &w.out[pod].status, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (status != NHD_NO_CANDIDATE) {
        memset(node_reason, NHD_WHY_NONE, (size_t)h->n_nodes);
        return NHD_OK;
    }
    int nf = 0;
    if ((rc = explain_prepare(h, w, &nf)) != NHD_OK) return rc;
    const int32_t one[1] = {pod};                    /* explain just this pod: failed[0] = pod, n_failed = 1 */
    const int32_t n1 = 1;
    CK(cudaMemcpyAsync(h->d_xpod + w.n_pods, one, 4, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_xsmall, &n1, 4, cudaMemcpyHostToDevice, h->stream));
    CK(h->d_xreasons.grow((size_t)h->n_nodes));
    if ((rc = explain_launch(h, w, h->d_snapshot, 1, nullptr, h->d_xreasons)) != NHD_OK) return rc;
    CK(cudaMemcpyAsync(node_reason, h->d_xreasons, (size_t)h->n_nodes, cudaMemcpyDeviceToHost, h->stream));
    return explain_survivors(h, "nhd_explain_pod");
}

/* ------------------------------------------------------------------ placement queries and plans */

/* the records a query or a plan reads: NHD_QUERY_MIRROR or NHD_QUERY_SNAPSHOT, the latter only while the hardware
 * classes (d_class, d_cls_fast, d_sigs: the mirror's) describe it, i.e. no load or update since the snapshot */
static int32_t source_records(nhd_handle* h, int32_t source, const char* what, const uint8_t** records)
{
    if (source != NHD_QUERY_MIRROR && source != NHD_QUERY_SNAPSHOT)
        return fail(h, NHD_ERR_INVALID, "%s source %d is neither NHD_QUERY_MIRROR nor NHD_QUERY_SNAPSHOT", what, source);
    if (!h->loaded) return fail(h, NHD_ERR_STATE, "nhd_%s_batch before nhd_load_nodes", what);
    if (source == NHD_QUERY_SNAPSHOT && (!h->have_snapshot || h->snap_rec_gen != h->rec_gen))
        return fail(h, NHD_ERR_STATE, "a snapshot %s needs nhd_snapshot with no nhd_load_nodes / nhd_update_nodes since", what);
    *records = source == NHD_QUERY_SNAPSHOT ? h->d_snapshot : h->d_nodes;
    return NHD_OK;
}

/*
 * Where each pod would go on its own, on the mirror or on the snapshot, with nothing written but the query's own
 * scratch: de-duplicate into pod types (as nhd_stage_batch), filter the whole cluster into the query's bitmaps and
 * summaries (fast_tables_kernel + filter_kernel, no sharding, no exchange), one warp per pod picks the node
 * (query_select_kernel), one thread per placed pod works out the mapping and the assignment (query_assign_kernel).
 */
extern "C" int32_t nhd_query_batch(nhd_handle* h, int32_t source, int32_t n_pods, const nhd_pod* pods, const double* now,
                                   nhd_binding* out)
{
    if (!h || n_pods < 0 || (n_pods > 0 && (!pods || !now || !out))) return NHD_ERR_INVALID;
    const uint8_t* nodes = nullptr;
    int32_t rc = source_records(h, source, "query", &nodes);
    if (rc != NHD_OK) return rc;
    if (n_pods == 0) return NHD_OK;
    Workspace& w = h->scratch;
    if ((rc = stage_pods(h, w, n_pods, pods, now, h->max_numa)) != NHD_OK) return rc;

    /* the candidate bitmaps of the query's pod types on the chosen records */
    if ((rc = launch_solve(h, w, nodes, false, false, true)) != NHD_OK) return rc;

    /* each pod on its own: the node, then the mapping and the assignment on a copy of its record */
    QueryArgs qa;
    qa.nodes = nodes; qa.types = w.types; qa.pod_type = w.pod_type(); qa.now = w.now();
    qa.bitmaps = w.bitmaps; qa.pod_groups = w.pod_groups(); qa.names_used = w.names_used;
    qa.out = w.out; qa.n_pods = n_pods; qa.n_types = w.n_types; qa.words = h->words;
    qa.min_busy = h->params.min_busy_secs;
    memcpy(qa.cap, h->cap, sizeof(qa.cap));
    const int warps_per_cta = QUERY_SELECT_THREADS / 32;
    query_select_kernel<<<(n_pods + warps_per_cta - 1) / warps_per_cta, QUERY_SELECT_THREADS, 0, h->stream>>>(qa);
    CK(cudaGetLastError());
    query_assign_kernel<<<(n_pods + 63) / 64, 64, 0, h->stream>>>(qa);
    CK(cudaGetLastError());
    return fetch_bindings(h, w, n_pods, out);
}

/*
 * The bindings nhd_solve_batch would return on the chosen records with the excluded nodes in maintenance, and
 * optionally nhd_explain_batch's counts after it, with nothing written but the scratch: the solve's own launches
 * (launch_solve) on the scratch workspace, without the commit and without sharding.  With exclusions the records are
 * first copied into a plan-owned array and the excluded nodes flagged there (exclude_nodes_kernel); without, the source
 * records are read in place.
 * With rounds (nhd_plan_batch_rounds, n_rounds > 0) the records are always copied, and every round but the last commits
 * to the copy; round r >= 1 is the same launches on the pods round r - 1 left unplaced, at round_clock[r - 1].  The pod
 * types are staged once; round_advance_kernel hands the unplaced pods (type, group mask, caller row) to the other half
 * of the double-buffered pod arrays and every binding to its caller's row, and the host reads one word per round, the
 * next round's pod count.  Only the last round can leave a NO_CANDIDATE last attempt (an unplaced pod is retried in
 * every round), so only it is explained, on the records it started from: it runs no commit.
 * With releases or tracked NIC counts (nhd_plan_batch_releases) release_kernel applies a round's releases to the copy
 * before its solve, and a round is solved in segments while a cut is still possible (the negative count the call can
 * hold, from its start and its releases so far, less the cuts made): each segment saves the records it starts from,
 * solves and commits, and claim_cut_kernel leaves the first pod that claimed a tracked NIC at <= -1 in the second
 * page-locked word.  On a cut the records are restored and the prefix up to that pod solved again with its commit; the
 * rest of the round is the next segment, at the same clock (Workspace::seg).  claim_count_kernel then adds the
 * segment's claims to the counts and clears the bits the counts leave at <= 0.  A last-round segment is explained on
 * the records it started from.
 * With arrivals (nhd_plan_batch_arrivals) every pod is staged once, arrivals included, and the staged arrays move to
 * d_apods, which no scan writes: round 0 and each run of a gap's arrivals (the arrivals between two release blocks, a
 * block being the gap's releases at or before the next arrival's clock) are solved from there as segments with their
 * commit, at their own clocks, cut as a round is.  arrival_advance_kernel then hands the gap's arrivals to its scan:
 * the failed ones behind the pods the previous scan left (whose count round_advance_kernel left in a device word, so
 * the host reads one word per gap).  With pod_clock every pod's clock starts as its own and round_clock_kernel writes
 * each scan's over the pods of the scan.
 */
static int32_t plan_batch(nhd_handle* h, const char* what, int32_t source, int32_t n_excluded, const int32_t* excluded,
                          int32_t n_pods, const nhd_pod* pods, const double* now, int32_t n_rounds,
                          const double* round_clock, int32_t n_tracked, const int32_t* tracked, const int16_t* pods_used,
                          int32_t n_releases, const nhd_release* releases, nhd_binding* out, uint32_t* why_counts,
                          int32_t* pod_round, const int32_t* arrive_round = nullptr, double* pod_clock = nullptr)
{
    if (!h || n_pods < 0 || n_excluded < 0 || (n_excluded > 0 && !excluded) || (n_pods > 0 && (!pods || !now || !out)))
        return NHD_ERR_INVALID;
    if (n_rounds < 0) return fail(h, NHD_ERR_INVALID, "%d rounds", n_rounds);
    if (n_rounds > 0 && !round_clock) return fail(h, NHD_ERR_INVALID, "%d rounds without round clocks", n_rounds);
    for (int r = 0; r < n_rounds; r++) {
        if (!std::isfinite(round_clock[r])) return fail(h, NHD_ERR_INVALID, "round clock %d is not finite", r);
        if (r > 0 && round_clock[r] < round_clock[r - 1]) return fail(h, NHD_ERR_INVALID, "round clocks go down at %d", r);
    }
    /* the clock rules read the pods pending at the start only: a monotonic clock never goes back */
    const auto at_start = [&](int i) { return !arrive_round || arrive_round[i] == 0; };
    for (int i = 0; i < n_pods && n_rounds > 0; i++)
        if (at_start(i) && round_clock[0] < now[i])
            return fail(h, NHD_ERR_INVALID, "round clock 0 is earlier than the clock of pod %d", i);
    if (n_tracked < 0 || n_releases < 0 || (n_tracked > 0 && (!tracked || !pods_used)) || (n_releases > 0 && !releases))
        return fail(h, NHD_ERR_INVALID, "%d tracked nodes, %d releases", n_tracked, n_releases);
    double t0 = -INFINITY;
    for (int i = 0; i < n_pods; i++) if (at_start(i)) t0 = std::max(t0, now[i]);
    /* arrivals (nhd_plan_batch_arrivals): rounds in [0, n_rounds] never going down in pod order, and each arrival's
     * clock inside its gap, not before the arrival before it in that gap.  first_of[g]: the first pod arriving in gap g
     * or later (first_of[0] = 0), so gap g's arrivals are [first_of[g], first_of[g + 1]) */
    std::vector<int> first_of((size_t)n_rounds + 2, n_pods);
    first_of[0] = 0;
    double t_start = -INFINITY;                                /* the latest clock of the round-0 pods so far */
    for (int i = 0; i < n_pods && arrive_round; i++) {
        const int g = arrive_round[i];
        if (g != 0 && n_rounds == 0) return fail(h, NHD_ERR_INVALID, "pod %d arrives without rounds", i);
        if (g < 0 || g > n_rounds) return fail(h, NHD_ERR_INVALID, "pod %d: arrival round %d outside [0, %d]", i, g, n_rounds);
        if (i > 0 && g < arrive_round[i - 1]) return fail(h, NHD_ERR_INVALID, "arrival rounds go down at pod %d", i);
        if (g == 0) { t_start = std::max(t_start, now[i]); continue; }
        if (i > 0 && g == arrive_round[i - 1] && now[i] < now[i - 1])
            return fail(h, NHD_ERR_INVALID, "arrival clocks go down at pod %d", i);
        if (now[i] < (g > 1 ? round_clock[g - 2] : t_start) || now[i] > round_clock[g - 1])
            return fail(h, NHD_ERR_INVALID, "pod %d: arrival clock outside the gap before round %d", i, g);
        for (int k = g; k >= 1 && first_of[k] == n_pods; k--) first_of[k] = i;
    }
    const bool arrivals = first_of[1] < n_pods;
    for (int k = 0; k < n_releases; k++) {
        const nhd_release& rl = releases[k];
        if (rl.round < 1 || rl.round > n_rounds)
            return fail(h, NHD_ERR_INVALID, "release %d: round %d outside [1, %d]", k, rl.round, n_rounds);
        if (!std::isfinite(rl.clock)) return fail(h, NHD_ERR_INVALID, "release %d: clock is not finite", k);
        if (k > 0 && rl.clock < releases[k - 1].clock) return fail(h, NHD_ERR_INVALID, "release clocks go down at %d", k);
        if (rl.clock < (rl.round > 1 ? round_clock[rl.round - 2] : t0) || rl.clock > round_clock[rl.round - 1])
            return fail(h, NHD_ERR_INVALID, "release %d: clock outside the gap before round %d", k, rl.round);
    }
    const uint8_t* records = nullptr;
    int32_t rc = source_records(h, source, "plan", &records);
    if (rc != NHD_OK) return rc;
    const bool track = n_tracked > 0 || n_releases > 0;

    /* the tracked nodes' slots, the releases grouped by block and node (array order kept), the counts; the checks that
     * need the records run on the device.  A block is the releases of one gap played between the same two solves:
     * those before arrival i of the gap (clock <= now[i], after the arrival before it), or after the gap's last arrival
     * and before its scan (i = first_of[round + 1]); without arrivals a round's releases are one block */
    struct RelBlock { int round, pod, g0, g1; long long pairs; };
    const int N = h->n_nodes, T = n_tracked, R = n_releases;
    std::vector<int32_t> rel_area;
    std::vector<RelBlock> blocks;
    long long neg0 = 0;
    size_t off_slot = 0, off_rslot = 0, off_nrel = 0, off_nstart = 0, off_bad = 0;
    if (track) {
        off_slot = (size_t)T * NHD_MAX_NICS; off_rslot = off_slot + N; off_nrel = off_rslot + R; off_nstart = off_nrel + R;
        rel_area.assign(off_nstart, 0);
        for (int t = 0; t < T; t++)
            for (int i = 0; i < NHD_MAX_NICS; i++) {
                const int c = pods_used[(size_t)t * NHD_MAX_NICS + i];
                rel_area[(size_t)t * NHD_MAX_NICS + i] = c;
                neg0 += c < 0 ? -c : 0;
            }
        int32_t* slot = rel_area.data() + off_slot;
        for (int n = 0; n < N; n++) slot[n] = -1;
        for (int t = 0; t < T; t++) {
            const int32_t n = tracked[t];
            if (n < 0 || n >= N) return fail(h, NHD_ERR_INVALID, "tracked node %d outside the %d loaded nodes", n, N);
            if (slot[n] >= 0) return fail(h, NHD_ERR_INVALID, "node %d tracked twice", n);
            slot[n] = t;
        }
        std::vector<int32_t> order((size_t)R), before((size_t)R);
        for (int k = 0; k < R; k++) {
            const int32_t n = releases[k].node;
            if (n < 0 || n >= N || slot[n] < 0) return fail(h, NHD_ERR_INVALID, "release %d: node %d is not tracked", k, n);
            rel_area[off_rslot + k] = slot[n];
            order[k] = k;
            const int g = releases[k].round;
            before[k] = (int32_t)(std::lower_bound(now + first_of[g], now + first_of[g + 1], releases[k].clock) - now);
        }
        std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) {
            return std::make_tuple(releases[a].round, before[a], slot[releases[a].node]) <
                   std::make_tuple(releases[b].round, before[b], slot[releases[b].node]);
        });
        for (int k = 0; k < R; k++) {
            rel_area[off_nrel + k] = order[k];
            const int a = order[k], p = k ? order[k - 1] : -1;
            const nhd_release& rl = releases[a];
            const bool new_block = k == 0 || rl.round != releases[p].round || before[a] != before[p];
            if (new_block) blocks.push_back({rl.round, before[a], 0, 0, 0});
            if (new_block || rl.node != releases[p].node) {
                blocks.back().g1++;
                rel_area.push_back(k);
            }
            for (int i = 0; i < NHD_MAX_NICS; i++) blocks.back().pairs += rl.nic_pairings[i];
        }
        rel_area.push_back(R);
        for (size_t b = 0, g = 0; b < blocks.size(); b++) {
            blocks[b].g0 = (int)g;
            g += blocks[b].g1;
            blocks[b].g1 = (int)g;
        }
        off_bad = rel_area.size();
        rel_area.push_back(0x7FFFFFFF);
        CK(cudaSetDevice(h->params.device));
        CK(h->d_rel.grow(rel_area.size() * 4));
        CK(h->d_rels.grow((size_t)std::max(R, 1) * sizeof(nhd_release)));
        CK(h->d_pidx.grow((size_t)std::max(T, 1) * (4 + NHD_MAX_NICS * 2)));
        CK(cudaMemcpyAsync(h->d_rel, rel_area.data(), rel_area.size() * 4, cudaMemcpyHostToDevice, h->stream));
        if (R) CK(cudaMemcpyAsync(h->d_rels, releases, (size_t)R * sizeof(nhd_release), cudaMemcpyHostToDevice, h->stream));
        if (T) {
            CK(cudaMemcpyAsync(h->d_pidx, tracked, (size_t)T * 4, cudaMemcpyHostToDevice, h->stream));
            CK(cudaMemcpyAsync(h->d_pidx + T, pods_used, (size_t)T * NHD_MAX_NICS * 2, cudaMemcpyHostToDevice, h->stream));
        }
        release_check_kernel<<<(R + T + 255) / 256, 256, 0, h->stream>>>(records, h->d_rels, R, h->d_pidx,
                                                                          reinterpret_cast<const int16_t*>(h->d_pidx + T), T,
                                                                          h->d_rel + off_bad);
        CK(cudaGetLastError());
        int32_t bad = 0;
        CK(cudaMemcpyAsync(&bad, h->d_rel + off_bad, 4, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        if (bad < R)
            return fail(h, NHD_ERR_INVALID, "release %d: a core, GPU or NIC beyond node %d's own", bad, releases[bad].node);
        if (bad != 0x7FFFFFFF)
            return fail(h, NHD_ERR_INVALID, "tracked node %d: pods_used disagrees with its NIC bits", tracked[bad - R]);
    }

    /* the excluded nodes, each once; the tuple limits are judged as the equivalent solve would, on the largest NUMA
     * count among the nodes the filter could accept once they are in maintenance */
    std::vector<int32_t> ex;
    int hist[NHD_MAX_NUMA + 1];
    memcpy(hist, h->numa_hist, sizeof(hist));
    {
        std::vector<uint8_t> seen((size_t)h->n_nodes, 0);
        for (int i = 0; i < n_excluded; i++) {
            const int32_t n = excluded[i];
            if (n < 0 || n >= h->n_nodes)
                return fail(h, NHD_ERR_INVALID, "excluded node %d outside the %d loaded nodes", n, h->n_nodes);
            if (seen[n]) continue;
            seen[n] = 1;
            ex.push_back(n);
            hist[h->node_numa[n]]--;
            hist[0]++;
        }
    }
    int max_numa = 1;
    for (int k = 2; k <= NHD_MAX_NUMA; k++) if (hist[k] > 0) max_numa = k;
    if (n_pods == 0) return NHD_OK;
    Workspace& w = h->scratch;
    if ((rc = stage_pods(h, w, n_pods, pods, now, max_numa)) != NHD_OK) return rc;
    const uint8_t* nodes = records;
    if (!ex.empty() || n_rounds > 0 || track) {
        CK(h->d_pnodes.grow(h->nodes_bytes));
        CK(cudaMemcpyAsync(h->d_pnodes, records, h->nodes_bytes, cudaMemcpyDeviceToDevice, h->stream));
        nodes = h->d_pnodes;
    }
    if (!ex.empty()) {
        CK(h->d_pidx.grow(ex.size() * 4));
        CK(cudaMemcpyAsync(h->d_pidx, ex.data(), ex.size() * 4, cudaMemcpyHostToDevice, h->stream));
        exclude_nodes_kernel<<<(unsigned)((ex.size() + 255) / 256), 256, 0, h->stream>>>(h->d_pnodes, h->d_pidx, (int)ex.size());
        CK(cudaGetLastError());
    }
    if (n_rounds == 0 && !track) {
        if (pod_round) memset(pod_round, 0, (size_t)n_pods * 4);
        if (pod_clock) memcpy(pod_clock, now, (size_t)n_pods * 8);
        if ((rc = launch_solve(h, w, nodes, false, false, false)) != NHD_OK) return rc;
        if (why_counts && (rc = explain_counts(h, w, nodes, why_counts, what)) != NHD_OK) return rc;
        return fetch_bindings(h, w, n_pods, out);
    }

    const size_t P = (size_t)n_pods, grid0 = (P + ROUND_THREADS - 1) / ROUND_THREADS, why_bytes = P * NHD_WHY_COUNT * 4;
    const size_t off_now = w.now_offset(), off_gm = off_now + P * 8, pods_bytes = off_gm + (w.n_names ? P * 8 : 0);
    CK(h->d_rpods.grow(pods_bytes));
    CK(h->d_ridx.grow((3 * P + grid0 + 1) * 4));
    CK(h->d_rout.grow(P * sizeof(nhd_binding)));
    CK(h->h_rcount.grow(8));
    if (why_counts) {
        CK(h->d_rwhy.grow(why_bytes));
        CK(cudaMemsetAsync(h->d_rwhy, 0, why_bytes, h->stream));
    }
    if (pod_clock) {            /* every pod's first attempt is at its own clock; each scan writes its clock over it */
        CK(h->d_rclock.grow(P * 8));
        CK(cudaMemcpyAsync(h->d_rclock, w.pod_arrays + off_now, P * 8, cudaMemcpyDeviceToDevice, h->stream));
    }
    if (arrivals) {
        /* round 0 and the arrival runs solve from the staged pods, kept in d_apods, where no scan's pod list is
         * written; the scans alternate between w.pod_arrays and d_rpods */
        CK(h->d_apods.grow(pods_bytes));
        w.pod_arrays.swap(h->d_apods);
    }
    const auto from_staged = [&]() { if (arrivals) w.pod_arrays.swap(h->d_apods); };   /* (called in pairs) */
    int32_t* const rows[2] = {h->d_ridx, h->d_ridx + P};
    int32_t* const d_base = h->d_ridx + 3 * P + grid0;    /* with arrivals: pods the last scan left, for the next gap */
    if (track) {
        /* round 0's caller rows are the pods' own (its reason rows are scattered per segment) */
        std::vector<int32_t> iota(P);
        for (size_t i = 0; i < P; i++) iota[i] = (int32_t)i;
        CK(cudaMemcpyAsync(rows[0], iota.data(), P * 4, cudaMemcpyHostToDevice, h->stream));
        CK(h->d_pseg.grow(h->nodes_bytes));
    }
    int32_t* const d_count = h->d_rel;
    const int32_t* const d_slot = h->d_rel + off_slot;
    uint8_t* const pnodes = h->d_pnodes;
    long long cut_room = neg0;                /* negative count the plan's copy may hold: an upper bound on cuts */
    size_t next_block = 0;

    /* the releases of gap r played right before arrival i (i = first_of[r + 1]: before the scan) */
    const auto play = [&](int r, int i) -> int32_t {
        for (; next_block < blocks.size() && blocks[next_block].round == r && blocks[next_block].pod == i; next_block++) {
            const RelBlock& b = blocks[next_block];
            ReleaseArgs rla;
            rla.nodes = pnodes; rla.rel = h->d_rels; rla.rel_slot = h->d_rel + off_rslot;
            rla.node_start = h->d_rel + off_nstart + b.g0; rla.node_rel = h->d_rel + off_nrel;
            rla.n = b.g1 - b.g0; rla.count = d_count;
            release_kernel<<<(rla.n + 127) / 128, 128, 0, h->stream>>>(rla);
            CK(cudaGetLastError());
            cut_room += b.pairs;
        }
        return NHD_OK;
    };
    /* pods [first, first + m) of w solved in order, committed unless this is the last scan, explained when asked (row:
     * the scan's caller rows).  With tracked counts: in segments while a cut is possible, each starting at its first
     * pod's own clock when per_pod (round 0 and the arrival runs), else at w.now0 */
    const auto solve = [&](int first, int m, bool commit, bool explain, int32_t* row, bool per_pod) -> int32_t {
        if (!track) {
            w.seg = first;
            w.n_pods = m;
            const int32_t e = launch_solve(h, w, nodes, false, commit, false);
            w.seg = 0;
            return e;
        }
        int32_t e;
        for (int seg = first; seg < first + m;) {
            w.seg = seg;
            w.n_pods = first + m - seg;
            if (per_pod) w.now0 = now[seg];
            if (cut_room <= 0) {
                /* no claim can meet a negative count: the rest of the run is one segment, as without releases */
                const int k = w.n_pods;
                nhd_binding* const b = w.bindings();
                if ((e = launch_solve(h, w, nodes, false, commit, false)) != NHD_OK) return e;
                if (commit) {
                    claim_count_kernel<<<(k + 127) / 128, 128, 0, h->stream>>>(b, k, d_slot, d_count, pnodes);
                    CK(cudaGetLastError());
                }
                if (explain) {
                    if ((e = explain_rows(h, w, nodes)) != NHD_OK) return e;
                    round_why_kernel<<<(k * NHD_WHY_COUNT + 255) / 256, 256, 0, h->stream>>>(h->d_xcounts, row + seg, k,
                                                                                             h->d_rwhy);
                    CK(cudaGetLastError());
                }
                break;
            }
            nhd_binding* const b = w.bindings();
            int32_t* const cut_word = h->h_rcount + 1;
            uint8_t* const seg_nodes = h->d_pseg;
            CK(cudaMemcpyAsync(seg_nodes, pnodes, h->nodes_bytes, cudaMemcpyDeviceToDevice, h->stream));
            if ((e = launch_solve(h, w, nodes, false, true, false)) != NHD_OK) return e;
            int k = w.n_pods;
            claim_cut_kernel<<<1, CUT_THREADS, 0, h->stream>>>(b, k, d_slot, d_count, cut_word);
            CK(cudaGetLastError());
            CK(cudaStreamSynchronize(h->stream));
            const int cut = *cut_word;
            if (cut >= 0) {
                CK(cudaMemcpyAsync(pnodes, seg_nodes, h->nodes_bytes, cudaMemcpyDeviceToDevice, h->stream));
                w.n_pods = k = cut + 1;
                if ((e = launch_solve(h, w, nodes, false, true, false)) != NHD_OK) return e;
                cut_room--;
            }
            claim_count_kernel<<<(k + 127) / 128, 128, 0, h->stream>>>(b, k, d_slot, d_count, pnodes);
            CK(cudaGetLastError());
            if (explain) {
                if ((e = explain_rows(h, w, seg_nodes)) != NHD_OK) return e;
                round_why_kernel<<<(k * NHD_WHY_COUNT + 255) / 256, 256, 0, h->stream>>>(h->d_xcounts, row + seg, k,
                                                                                         h->d_rwhy);
                CK(cudaGetLastError());
                if ((e = explain_survivors(h, what)) != NHD_OK) return e;
            }
            seg += k;
        }
        w.seg = 0;
        return NHD_OK;
    };

    RoundArgs ra;
    ra.result = h->d_rout; ra.pod_round = h->d_ridx + 2 * P; ra.block_cnt = h->d_ridx + 3 * P;
    ra.n_rounds = n_rounds;
    /* n: the pods of the next scan, -1 while only the device knows it (the gap's hand-over reads it there) */
    int n = first_of[1], cur = 0;
    for (int r = 0; r <= n_rounds && (n != 0 || first_of[r] < n_pods); r++) {
        const bool last = r == n_rounds;
        if (r > 0) {
            /* gap r: its releases and the runs of its arrivals between them, merged by clock, then the hand-over of
             * the arrivals to scan r, behind the pods scan r - 1 left */
            for (int i = first_of[r], end = first_of[r + 1];; ) {
                if ((rc = play(r, i)) != NHD_OK) return rc;
                if (i == end) break;
                const int j = next_block < blocks.size() && blocks[next_block].round == r ? blocks[next_block].pod : end;
                w.now0 = now[i];
                w.const_clock = now[i] == now[j - 1];
                from_staged();
                rc = solve(i, j - i, true, false, nullptr, true);
                from_staged();
                if (rc != NHD_OK) return rc;
                i = j;
            }
            if (first_of[r] < n_pods) {             /* scan r - 1 deferred its count to this hand-over */
                const int a0 = first_of[r], m = first_of[r + 1] - a0, grid = std::max(1, (m + ROUND_THREADS - 1) / ROUND_THREADS);
                RoundArgs rc_args = ra;
                rc_args.out = w.out + a0; rc_args.n_pods = m;
                round_count_kernel<<<grid, ROUND_THREADS, 0, h->stream>>>(rc_args);
                ArrivalArgs aa;
                from_staged();
                aa.out = w.out + a0; aa.pod_type = w.pod_type() + a0; aa.now = w.now() + a0;
                aa.pod_groups = w.n_names ? w.pod_groups() + a0 : nullptr;
                from_staged();
                aa.first = a0; aa.n_pods = m; aa.round = r; aa.n_rounds = n_rounds;
                aa.result = h->d_rout; aa.pod_round = ra.pod_round; aa.pod_clock = pod_clock ? h->d_rclock.p : nullptr;
                aa.block_cnt = ra.block_cnt; aa.base = d_base;
                aa.next_pod_type = reinterpret_cast<int32_t*>(w.pod_arrays.p);
                aa.next_now = reinterpret_cast<double*>(w.pod_arrays.p + off_now);
                aa.next_pod_groups = w.n_names ? reinterpret_cast<uint64_t*>(w.pod_arrays.p + off_gm) : nullptr;
                aa.next_row = rows[cur]; aa.next_clock = round_clock[r - 1]; aa.count = h->h_rcount;
                arrival_advance_kernel<<<grid, ROUND_THREADS, 0, h->stream>>>(aa);
                CK(cudaGetLastError());
                CK(cudaStreamSynchronize(h->stream));
                n = *h->h_rcount;
            }
        }
        /* scan r (round 0: the pods pending at the start, at their own clocks) */
        const bool defer = !last && first_of[r + 1] < n_pods;      /* the next gap's hand-over reads the count */
        if (n > 0) {
            w.seg = 0;
            w.n_pods = n;
            if (r > 0) { w.now0 = round_clock[r - 1]; w.const_clock = true; }
            else {
                w.now0 = now[0];
                w.const_clock = true;
                for (int i = 1; i < n; i++) if (now[i] != now[0]) { w.const_clock = false; break; }
            }
            int32_t* const row = r || track ? rows[cur] : nullptr;
            if (r == 0) from_staged();
            if ((rc = solve(0, n, !last, last && why_counts, row, r == 0)) != NHD_OK) { if (r == 0) from_staged(); return rc; }
            ra.out = w.out; ra.pod_type = w.pod_type(); ra.pod_groups = w.pod_groups(); ra.row = row;
            ra.n_pods = n; ra.round = r;
            ra.next_pod_type = last ? nullptr : reinterpret_cast<int32_t*>(h->d_rpods.p);
            ra.next_now = last ? nullptr : reinterpret_cast<double*>(h->d_rpods.p + off_now);
            ra.next_pod_groups = last || !w.n_names ? nullptr : reinterpret_cast<uint64_t*>(h->d_rpods.p + off_gm);
            ra.next_row = last ? nullptr : rows[cur ^ 1];
            ra.next_clock = last ? 0.0 : round_clock[r];
            ra.survivors = defer ? d_base : h->h_rcount.p;
            const int grid = (n + ROUND_THREADS - 1) / ROUND_THREADS;
            if (!last) round_count_kernel<<<grid, ROUND_THREADS, 0, h->stream>>>(ra);
            round_advance_kernel<<<grid, ROUND_THREADS, 0, h->stream>>>(ra);
            CK(cudaGetLastError());
            if (pod_clock && r > 0) {
                round_clock_kernel<<<(n + 255) / 256, 256, 0, h->stream>>>(row, n, round_clock[r - 1], h->d_rclock);
                CK(cudaGetLastError());
            }
            if (r == 0) from_staged();
            if (last) {
                if (why_counts && !track) {
                    if ((rc = explain_rows(h, w, nodes)) != NHD_OK) return rc;
                    round_why_kernel<<<(n * NHD_WHY_COUNT + 255) / 256, 256, 0, h->stream>>>(h->d_xcounts, ra.row, n, h->d_rwhy);
                    CK(cudaGetLastError());
                }
                break;
            }
        } else if (defer) {
            CK(cudaMemsetAsync(d_base, 0, 4, h->stream));
        }
        if (last) break;
        if (defer) {
            n = -1;
        } else if (n > 0) {
            CK(cudaStreamSynchronize(h->stream));
            n = *h->h_rcount;
        }
        w.pod_arrays.swap(h->d_rpods);
        cur ^= 1;
    }
    if (why_counts) CK(cudaMemcpyAsync(why_counts, h->d_rwhy, why_bytes, cudaMemcpyDeviceToHost, h->stream));
    if (pod_round) CK(cudaMemcpyAsync(pod_round, ra.pod_round, P * 4, cudaMemcpyDeviceToHost, h->stream));
    if (pod_clock) CK(cudaMemcpyAsync(pod_clock, h->d_rclock, P * 8, cudaMemcpyDeviceToHost, h->stream));
    if ((rc = fetch_bindings(h, w, n_pods, out, h->d_rout)) != NHD_OK) return rc;
    return why_counts && n > 0 ? explain_survivors(h, what) : NHD_OK;
}

extern "C" int32_t nhd_plan_batch(nhd_handle* h, int32_t source, int32_t n_excluded, const int32_t* excluded,
                                  int32_t n_pods, const nhd_pod* pods, const double* now, nhd_binding* out,
                                  uint32_t* why_counts)
{
    return plan_batch(h, "nhd_plan_batch", source, n_excluded, excluded, n_pods, pods, now, 0, nullptr, 0, nullptr,
                      nullptr, 0, nullptr, out, why_counts, nullptr);
}

extern "C" int32_t nhd_plan_batch_rounds(nhd_handle* h, int32_t source, int32_t n_excluded, const int32_t* excluded,
                                         int32_t n_pods, const nhd_pod* pods, const double* now, int32_t n_rounds,
                                         const double* round_clock, nhd_binding* out, uint32_t* why_counts,
                                         int32_t* pod_round)
{
    return plan_batch(h, "nhd_plan_batch_rounds", source, n_excluded, excluded, n_pods, pods, now, n_rounds, round_clock,
                      0, nullptr, nullptr, 0, nullptr, out, why_counts, pod_round);
}

extern "C" int32_t nhd_plan_batch_releases(nhd_handle* h, int32_t source, int32_t n_excluded, const int32_t* excluded,
                                           int32_t n_pods, const nhd_pod* pods, const double* now, int32_t n_rounds,
                                           const double* round_clock, int32_t n_tracked, const int32_t* tracked,
                                           const int16_t* pods_used, int32_t n_releases, const nhd_release* releases,
                                           nhd_binding* out, uint32_t* why_counts, int32_t* pod_round)
{
    return plan_batch(h, "nhd_plan_batch_releases", source, n_excluded, excluded, n_pods, pods, now, n_rounds,
                      round_clock, n_tracked, tracked, pods_used, n_releases, releases, out, why_counts, pod_round);
}

extern "C" int32_t nhd_plan_batch_arrivals(nhd_handle* h, int32_t source, int32_t n_excluded, const int32_t* excluded,
                                           int32_t n_pods, const nhd_pod* pods, const double* now, int32_t n_rounds,
                                           const double* round_clock, int32_t n_tracked, const int32_t* tracked,
                                           const int16_t* pods_used, int32_t n_releases, const nhd_release* releases,
                                           const int32_t* arrive_round, nhd_binding* out, uint32_t* why_counts,
                                           int32_t* pod_round, double* pod_clock)
{
    return plan_batch(h, "nhd_plan_batch_arrivals", source, n_excluded, excluded, n_pods, pods, now, n_rounds,
                      round_clock, n_tracked, tracked, pods_used, n_releases, releases, out, why_counts, pod_round,
                      arrive_round, pod_clock);
}

/*
 * Many independent plans at once, each on the source records with its own excluded nodes and its own replaced records:
 * every scenario's pods are checked as nhd_stage_batch checks them (a refusal refuses that scenario only), the pods of
 * the accepted scenarios are de-duplicated into one pod set and filtered once on the unchanged source records
 * (launch_solve's tables + filter, as a query), then one warp per scenario walks its pods in order
 * (scenario_plan_kernel), starting from its edited records and lifting its exclusions at its lift index.  The tuple
 * limits are judged against the whole cluster's NUMA counts and those of the edit and added records: the shared filter
 * enumerates the tuples of every node, the excluded ones included, and an edited or added node is evaluated on its own
 * record.  Added nodes (nhd_plan_scenarios_grown) live only in the working slots, after the edited ones; a binding on
 * one names it n_nodes + its call-wide index.  With rounds (nhd_plan_scenarios_rounds) the same warp walks the
 * scenario's unplaced pods again at each round clock (scenario_plan_kernel<., true>); scenario s's slots then start at
 * slot_start[s] and hold n_edits + n_adds + min(n_s * (1 + R_s), n_nodes) records, and the reasons' base pass reads
 * each pod's clock of its last attempt instead of the staged clocks.  With releases (nhd_plan_scenarios_releases,
 * scenario_plan_kernel<., true, true>, the rounds layout even without round clocks) the accepted scenarios' tracked
 * nodes, counts (int32, seeded from pods_used, after the pod rounds in d_sidx) and releases are compacted like the
 * rest, each release carrying its node's compacted count row; a scenario's slots grow by its distinct released nodes,
 * min(n_s * (1 + R_s) + D_s, n_nodes).  release_check_kernel first checks the call's releases and tracked counts
 * against the source records, one word read back.  With arrivals (nhd_plan_scenarios_arrivals,
 * scenario_plan_kernel<., true, true, true>, the releases' layout even without releases) each timeline is expanded
 * into the kernel's rounds, each over its own pod range (round 0, one round per arrival at its clock, one per scan
 * over the pods arrived so far), each release attached to the round it precedes; pod_round is mapped back to the
 * call's rounds, and pod_clock is the clock of each pod's last kernel round.
 */
/*
 * why_counts of the scenario call just run on w (its bindings b, its pods and clocks run_pods / run_now, its correction
 * rows in d_xpod + 2 * n_run; with rounds, run_now and its device copy d_now are the clocks of each pod's last attempt,
 * else d_now is null and the staged clocks serve): the NO_CANDIDATE pods' keys (pod type, clock, node-group mask) de-duplicated, one
 * explain_kernel pass per key over the source records with no bindings (empty per-node lists), then
 * scenario_why_combine_kernel adds each pod's correction to its key's row.  rows: n_run * NHD_WHY_COUNT host entries.
 * Buffers were sized before the scenario kernel; one host wait.
 */
static int32_t scenario_reasons(nhd_handle* h, const Workspace& w, const uint8_t* records, int n_run,
                                const nhd_pod* run_pods, const double* run_now, const double* d_now,
                                const nhd_binding* b, uint32_t* rows, const char* what)
{
    const int N = h->n_nodes;
    std::vector<int32_t> idx(2 * (size_t)n_run, -1);              /* base_row | key representatives */
    std::map<std::tuple<int32_t, uint64_t, uint64_t>, int32_t> keys;
    int n_keys = 0;
    for (int i = 0; i < n_run; i++) {
        if (b[i].status != NHD_NO_CANDIDATE) continue;
        uint64_t clock;
        memcpy(&clock, &run_now[i], 8);
        const auto it = keys.emplace(std::make_tuple(w.pod_type_host[i], clock, w.n_names ? run_pods[i].group_mask : 0), i).first;
        if (it->second == i) idx[(size_t)n_run + n_keys++] = i;
        idx[i] = it->second;
    }
    if (n_keys == 0) {
        memset(rows, 0, (size_t)n_run * NHD_WHY_COUNT * 4);
        return NHD_OK;
    }
    uint32_t* base = h->d_xcounts;
    uint32_t* d_rows = h->d_xcounts + (size_t)n_run * NHD_WHY_COUNT;
    const int32_t small[4] = {n_keys, 0, 0, 0};                  /* n_failed (keys), survivors, bad */
    CK(cudaMemcpyAsync(h->d_xpod, idx.data(), idx.size() * 4, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_xsmall, small, 16, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemsetAsync(h->d_xnode + N, 0, ((size_t)N + 1) * 4, h->stream));
    CK(cudaMemsetAsync(base, 0, (size_t)n_run * NHD_WHY_COUNT * 4, h->stream));
    /* the key's row on the source records: the representative pod with nothing bound before it; nodes that pass
     * every stage land in survivors, which is not read (pass bucket = n_nodes - row sum) */
    int32_t rc = explain_launch(h, w, records, n_keys, base, nullptr, d_now);
    if (rc != NHD_OK) return rc;
    scenario_why_combine_kernel<<<(unsigned)((n_run + 255) / 256), 256, 0, h->stream>>>(
        base, h->d_xpod, h->d_xpod + 2 * (size_t)n_run, n_run, N, d_rows, h->d_xsmall + 2);
    CK(cudaGetLastError());
    uint32_t bad = 0;
    CK(cudaMemcpyAsync(rows, d_rows, (size_t)n_run * NHD_WHY_COUNT * 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(&bad, h->d_xsmall + 2, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (bad) return fail(h, NHD_ERR_STATE, "%s: %u NO_CANDIDATE rows with a negative bucket or a node passing every stage",
                         what, bad);
    return NHD_OK;
}

static int32_t plan_scenarios(nhd_handle* h, const char* what, int32_t source, int32_t n_scenarios,
                              const int32_t* excl_start, const int32_t* excluded, const int32_t* lift_at,
                              const int32_t* edit_start, const int32_t* edit_node, const nhd_node_rec* edit_rec,
                              const int32_t* add_start, const int32_t* add_at, const nhd_node_rec* add_rec,
                              const int32_t* pod_start, const nhd_pod* pods, const double* now,
                              const int32_t* round_start, const double* round_clock, const int32_t* track_start,
                              const int32_t* tracked, const int16_t* pods_used, const int32_t* rel_start,
                              const nhd_release* releases, nhd_binding* out, int32_t* scenario_status,
                              int32_t* scenario_pod, uint32_t* why_counts, int32_t* pod_round,
                              const int32_t* arrive_round = nullptr, double* pod_clock = nullptr)
{
    if (!h || n_scenarios < 0 || !excl_start || !pod_start || (n_scenarios > 0 && (!scenario_status || !scenario_pod)))
        return NHD_ERR_INVALID;
    if (excl_start[0] != 0 || pod_start[0] != 0 || (edit_start && edit_start[0] != 0) || (add_start && add_start[0] != 0) ||
        (round_start && round_start[0] != 0) || (track_start && track_start[0] != 0) || (rel_start && rel_start[0] != 0))
        return fail(h, NHD_ERR_INVALID, "scenario offsets must start at 0");
    for (int s = 0; s < n_scenarios; s++)
        if (excl_start[s + 1] < excl_start[s] || pod_start[s + 1] < pod_start[s] ||
            (edit_start && edit_start[s + 1] < edit_start[s]) || (add_start && add_start[s + 1] < add_start[s]) ||
            (round_start && round_start[s + 1] < round_start[s]) || (track_start && track_start[s + 1] < track_start[s]) ||
            (rel_start && rel_start[s + 1] < rel_start[s]))
            return fail(h, NHD_ERR_INVALID, "scenario %d: offsets go down", s);
    const int n_excl = excl_start[n_scenarios], n_pods = pod_start[n_scenarios];
    const int n_edit = edit_start ? edit_start[n_scenarios] : 0, n_add = add_start ? add_start[n_scenarios] : 0;
    const int n_round = round_start ? round_start[n_scenarios] : 0;
    const int n_trk = track_start ? track_start[n_scenarios] : 0, n_rel = rel_start ? rel_start[n_scenarios] : 0;
    if ((n_excl > 0 && !excluded) || (n_pods > 0 && (!pods || !now || !out)) || (n_edit > 0 && (!edit_node || !edit_rec)) ||
        (n_add > 0 && (!add_at || !add_rec)) || (n_round > 0 && !round_clock) ||
        (n_trk > 0 && (!tracked || !pods_used)) || (n_rel > 0 && !releases))
        return NHD_ERR_INVALID;
    for (int s = 0; s < n_scenarios && n_round > 0; s++)
        for (int r = round_start[s]; r < round_start[s + 1]; r++) {
            if (!std::isfinite(round_clock[r]))
                return fail(h, NHD_ERR_INVALID, "scenario %d: round clock %d is not finite", s, r);
            if (r > round_start[s] && round_clock[r] < round_clock[r - 1])
                return fail(h, NHD_ERR_INVALID, "scenario %d: round clocks go down at %d", s, r);
            if (r == round_start[s])                     /* a monotonic clock never goes back */
                for (int i = pod_start[s]; i < pod_start[s + 1]; i++)
                    if ((!arrive_round || arrive_round[i] == 0) && round_clock[r] < now[i])
                        return fail(h, NHD_ERR_INVALID, "scenario %d: round clock %d is earlier than the clock of pod %d",
                                    s, r, i - pod_start[s]);
        }
    /* arrivals (nhd_plan_scenarios_arrivals): rounds in [0, R_s] never going down in pod order, and each arrival's
     * clock inside its gap, not before the arrival before it in that gap */
    for (int s = 0; s < n_scenarios && arrive_round; s++) {
        const int R_s = round_start ? round_start[s + 1] - round_start[s] : 0;
        const double* clk = round_start ? round_clock + round_start[s] : nullptr;
        double t0 = -INFINITY;                                         /* the latest clock of the round-0 pods */
        for (int i = pod_start[s]; i < pod_start[s + 1]; i++) {
            const int g = arrive_round[i], k = i - pod_start[s];
            if (g != 0 && R_s == 0) return fail(h, NHD_ERR_INVALID, "scenario %d: pod %d arrives without rounds", s, k);
            if (g < 0 || g > R_s)
                return fail(h, NHD_ERR_INVALID, "scenario %d: pod %d: arrival round %d outside [0, %d]", s, k, g, R_s);
            if (i > pod_start[s] && g < arrive_round[i - 1])
                return fail(h, NHD_ERR_INVALID, "scenario %d: arrival rounds go down at pod %d", s, k);
            if (g == 0) { t0 = std::max(t0, now[i]); continue; }
            if (i > pod_start[s] && g == arrive_round[i - 1] && now[i] < now[i - 1])
                return fail(h, NHD_ERR_INVALID, "scenario %d: arrival clocks go down at pod %d", s, k);
            if (now[i] < (g > 1 ? clk[g - 2] : t0) || now[i] > clk[g - 1])
                return fail(h, NHD_ERR_INVALID, "scenario %d: pod %d: arrival clock outside the gap before round %d", s,
                            k, g);
        }
    }
    if (pod_round && !round_start && n_pods > 0) memset(pod_round, 0, (size_t)n_pods * 4);
    const uint8_t* records = nullptr;
    int32_t rc = source_records(h, source, "plan", &records);
    if (rc != NHD_OK) return rc;
    for (int e = 0; e < n_excl; e++)
        if (excluded[e] < 0 || excluded[e] >= h->n_nodes)
            return fail(h, NHD_ERR_INVALID, "excluded node %d outside the %d loaded nodes", excluded[e], h->n_nodes);
    int max_numa = h->max_numa;
    for (int e = 0; e < n_edit; e++) {
        if (edit_node[e] < 0 || edit_node[e] >= h->n_nodes)
            return fail(h, NHD_ERR_INVALID, "edited node %d outside the %d loaded nodes", edit_node[e], h->n_nodes);
        if (nhd_validate_node(&edit_rec[e]) != NHD_OK)
            return fail(h, NHD_ERR_INVALID, "edit record %d rejected by nhd_validate_node", e);
        max_numa = std::max(max_numa, (int)edit_rec[e].n_numa);
    }
    for (int s = 0; s < n_scenarios && n_edit > 0; s++) {
        std::vector<int32_t> nodes(edit_node + edit_start[s], edit_node + edit_start[s + 1]);
        std::sort(nodes.begin(), nodes.end());
        if (std::adjacent_find(nodes.begin(), nodes.end()) != nodes.end())
            return fail(h, NHD_ERR_INVALID, "scenario %d: node %d edited twice", s, *std::adjacent_find(nodes.begin(), nodes.end()));
    }
    for (int s = 0; s < n_scenarios && lift_at; s++)
        if (lift_at[s] < 0 || lift_at[s] > pod_start[s + 1] - pod_start[s])
            return fail(h, NHD_ERR_INVALID, "scenario %d: lift index %d outside [0, %d]", s, lift_at[s],
                        pod_start[s + 1] - pod_start[s]);
    for (int s = 0; s < n_scenarios && lift_at && arrive_round; s++) {    /* lifted after round 0, or held throughout */
        int n0 = 0;
        while (pod_start[s] + n0 < pod_start[s + 1] && arrive_round[pod_start[s] + n0] == 0) n0++;
        if (lift_at[s] > n0 && lift_at[s] != pod_start[s + 1] - pod_start[s])
            return fail(h, NHD_ERR_INVALID, "scenario %d: lift index %d neither at most the %d pods of round 0 nor %d",
                        s, lift_at[s], n0, pod_start[s + 1] - pod_start[s]);
    }
    for (int s = 0; s < n_scenarios && n_add > 0; s++)
        for (int e = add_start[s]; e < add_start[s + 1]; e++) {
            if (add_at[e] < 0 || add_at[e] > h->n_nodes)
                return fail(h, NHD_ERR_INVALID, "added node %d: position %d outside [0, %d]", e, add_at[e], h->n_nodes);
            if (e > add_start[s] && add_at[e] < add_at[e - 1])
                return fail(h, NHD_ERR_INVALID, "scenario %d: added node positions go down at %d", s, e);
            if (nhd_validate_node(&add_rec[e]) != NHD_OK)
                return fail(h, NHD_ERR_INVALID, "added record %d rejected by nhd_validate_node", e);
            /* the handle holds capacities for its own speed classes only */
            for (int k = 0; k < add_rec[e].n_nics; k++)
                if (nic_speed_class(add_rec[e], k) >= h->params.n_speed_classes)
                    return fail(h, NHD_ERR_INVALID, "added record %d: NIC %d has speed class %d, the handle has %d", e,
                                k, nic_speed_class(add_rec[e], k), h->params.n_speed_classes);
            max_numa = std::max(max_numa, (int)add_rec[e].n_numa);
        }
    /* releases (nhd_plan_scenarios_releases): per release its node's call-wide tracked row, per scenario its distinct
     * released nodes (the slot bound grows by them) */
    const bool arrivals = arrive_round != nullptr;                     /* always with the releases' layout */
    const bool with_releases = track_start || rel_start || arrivals;
    std::vector<int32_t> rel_row((size_t)n_rel), rel_nodes(with_releases ? n_scenarios : 0, 0);
    for (int s = 0; s < n_scenarios && with_releases; s++) {
        const int t0 = track_start ? track_start[s] : 0, t1 = track_start ? track_start[s + 1] : 0;
        std::vector<std::pair<int32_t, int32_t>> trk;                   /* (node, call-wide row), sorted by node */
        for (int t = t0; t < t1; t++) {
            if (tracked[t] < 0 || tracked[t] >= h->n_nodes)
                return fail(h, NHD_ERR_INVALID, "tracked node %d outside the %d loaded nodes", tracked[t], h->n_nodes);
            trk.emplace_back(tracked[t], t);
        }
        std::sort(trk.begin(), trk.end());
        for (size_t k = 1; k < trk.size(); k++)
            if (trk[k].first == trk[k - 1].first)
                return fail(h, NHD_ERR_INVALID, "scenario %d: node %d tracked twice", s, trk[k].first);
        const int l0 = rel_start ? rel_start[s] : 0, l1 = rel_start ? rel_start[s + 1] : 0;
        const int R_s = round_start ? round_start[s + 1] - round_start[s] : 0;
        const double* clk = round_start ? round_clock + round_start[s] : nullptr;
        if (l1 > l0 && R_s == 0) return fail(h, NHD_ERR_INVALID, "scenario %d: releases without rounds", s);
        double t_first = -INFINITY;
        for (int i = pod_start[s]; i < pod_start[s + 1]; i++)
            if (!arrive_round || arrive_round[i] == 0) t_first = std::max(t_first, now[i]);
        std::vector<int32_t> seen;
        for (int k = l0; k < l1; k++) {
            const nhd_release& rl = releases[k];
            if (rl.round < 1 || rl.round > R_s)
                return fail(h, NHD_ERR_INVALID, "scenario %d: release %d: round %d outside [1, %d]", s, k - l0, rl.round, R_s);
            if (!std::isfinite(rl.clock))
                return fail(h, NHD_ERR_INVALID, "scenario %d: release %d: clock is not finite", s, k - l0);
            if (k > l0 && rl.clock < releases[k - 1].clock)
                return fail(h, NHD_ERR_INVALID, "scenario %d: release clocks go down at %d", s, k - l0);
            if (rl.clock < (rl.round > 1 ? clk[rl.round - 2] : t_first) || rl.clock > clk[rl.round - 1])
                return fail(h, NHD_ERR_INVALID, "scenario %d: release %d: clock outside the gap before round %d", s,
                            k - l0, rl.round);
            const auto it = std::lower_bound(trk.begin(), trk.end(), std::make_pair(rl.node, (int32_t)INT32_MIN));
            if (it == trk.end() || it->first != rl.node)
                return fail(h, NHD_ERR_INVALID, "scenario %d: release %d: node %d is not tracked", s, k - l0, rl.node);
            for (int e = edit_start ? edit_start[s] : 0; e < (edit_start ? edit_start[s + 1] : 0); e++)
                if (edit_node[e] == rl.node)
                    return fail(h, NHD_ERR_INVALID, "scenario %d: release %d: node %d is one the scenario edits", s,
                                k - l0, rl.node);
            rel_row[k] = it->second;
            seen.push_back(rl.node);
        }
        std::sort(seen.begin(), seen.end());
        rel_nodes[s] = (int32_t)(std::unique(seen.begin(), seen.end()) - seen.begin());
    }
    if (n_rel + n_trk > 0) {           /* the checks that need the records (release_check_kernel), one word read back */
        const int32_t none = 0x7FFFFFFF;
        CK(cudaSetDevice(h->params.device));
        CK(h->d_rel.grow(4));
        CK(h->d_rels.grow((size_t)std::max(n_rel, 1) * sizeof(nhd_release)));
        CK(h->d_pidx.grow((size_t)std::max(n_trk, 1) * (4 + NHD_MAX_NICS * 2)));
        CK(cudaMemcpyAsync(h->d_rel, &none, 4, cudaMemcpyHostToDevice, h->stream));
        if (n_rel) CK(cudaMemcpyAsync(h->d_rels, releases, (size_t)n_rel * sizeof(nhd_release), cudaMemcpyHostToDevice, h->stream));
        if (n_trk) {
            CK(cudaMemcpyAsync(h->d_pidx, tracked, (size_t)n_trk * 4, cudaMemcpyHostToDevice, h->stream));
            CK(cudaMemcpyAsync(h->d_pidx + n_trk, pods_used, (size_t)n_trk * NHD_MAX_NICS * 2, cudaMemcpyHostToDevice, h->stream));
        }
        release_check_kernel<<<(n_rel + n_trk + 255) / 256, 256, 0, h->stream>>>(
            records, h->d_rels, n_rel, h->d_pidx, reinterpret_cast<const int16_t*>(h->d_pidx + n_trk), n_trk, h->d_rel);
        CK(cudaGetLastError());
        int32_t bad = 0;
        CK(cudaMemcpyAsync(&bad, h->d_rel, 4, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        if (bad < n_rel)
            return fail(h, NHD_ERR_INVALID, "release %d: a core, GPU or NIC beyond node %d's own", bad, releases[bad].node);
        if (bad != none)
            return fail(h, NHD_ERR_INVALID, "tracked node %d: pods_used disagrees with its NIC bits", tracked[bad - n_rel]);
    }
    const bool rounds = round_start != nullptr || with_releases;

    /* per scenario: its refusal, or its place among the accepted ones (pods, exclusions and edits compacted, the
     * exclusions sorted and each once).  idx = pod offsets | exclusion offsets | exclusions | edit offsets | edited
     * nodes | lift indices | add offsets | add positions of the accepted scenarios, and with rounds | round offsets |
     * first working slots, and with releases | track offsets | tracked nodes | release offsets | release rows. */
    std::vector<int32_t> acc, pod_off{0}, ex_off{0}, ex, ed_off{0}, ed_node, lift, ad_off{0}, ad_at, rd_off{0}, sl_start;
    std::vector<int32_t> tr_off, tr_node, tr_count, rl_off, rl_row;
    std::vector<nhd_node_rec> ed_rec, ad_rec;
    std::vector<nhd_release> rl_rec;
    std::vector<double> rd_clock;
    /* with arrivals: per kernel round (n_rounds + 1 per accepted scenario) its pods [q0, q1) and the round r of the
     * call it belongs to; per release the kernel round it precedes */
    std::vector<int32_t> rd_pods, rd_ext, rel_iround(arrivals ? n_rel : 0);
    if (with_releases) { tr_off.push_back(0); rl_off.push_back(0); }
    size_t n_slots = 0;
    for (int s = 0; s < n_scenarios; s++) {
        scenario_status[s] = NHD_OK;
        scenario_pod[s] = -1;
        for (int i = pod_start[s]; i < pod_start[s + 1]; i++) {
            const int32_t v = check_pod(nullptr, i - pod_start[s], pods[i], now[i], max_numa);
            if (v != NHD_OK) { scenario_status[s] = v; scenario_pod[s] = i - pod_start[s]; break; }
        }
        if (scenario_status[s] != NHD_OK) continue;
        acc.push_back(s);
        pod_off.push_back(pod_off.back() + pod_start[s + 1] - pod_start[s]);
        const size_t e0 = ex.size();
        ex.insert(ex.end(), excluded + excl_start[s], excluded + excl_start[s + 1]);
        std::sort(ex.begin() + e0, ex.end());
        ex.erase(std::unique(ex.begin() + e0, ex.end()), ex.end());
        ex_off.push_back((int32_t)ex.size());
        if (n_edit > 0) {
            ed_node.insert(ed_node.end(), edit_node + edit_start[s], edit_node + edit_start[s + 1]);
            ed_rec.insert(ed_rec.end(), edit_rec + edit_start[s], edit_rec + edit_start[s + 1]);
        }
        ed_off.push_back((int32_t)ed_node.size());
        lift.push_back(lift_at ? lift_at[s] : pod_start[s + 1] - pod_start[s]);
        if (n_add > 0) {
            ad_at.insert(ad_at.end(), add_at + add_start[s], add_at + add_start[s + 1]);
            ad_rec.insert(ad_rec.end(), add_rec + add_start[s], add_rec + add_start[s + 1]);
        }
        ad_off.push_back((int32_t)ad_at.size());
        const int64_t n_s = pod_start[s + 1] - pod_start[s];
        int64_t touches = n_s;                 /* without rounds: one slot per pod, as scenario_plan_kernel<., false> */
        if (rounds) {
            const int64_t R_s = round_start ? round_start[s + 1] - round_start[s] : 0;
            if (arrivals) {
                /* the timeline as the kernel's rounds: round 0 over the pods pending at the start; then per gap g, in
                 * clock order, each arrival alone at its own clock (the gap's releases at or before that clock go
                 * first), and the scan over the pods arrived so far, after the gap's remaining releases */
                const int c0 = pod_off[pod_off.size() - 2], p0 = pod_start[s], p1 = pod_start[s + 1];
                const int l0 = rel_start ? rel_start[s] : 0, l1 = rel_start ? rel_start[s + 1] : 0;
                const int32_t e0 = (int32_t)rd_ext.size();                /* this scenario's round 0 */
                int i = p0;
                while (i < p1 && arrive_round[i] == 0) i++;
                rd_pods.insert(rd_pods.end(), {c0, c0 + i - p0});
                rd_ext.push_back(0);
                for (int g = 1; g <= R_s; g++) {
                    int k = l0;
                    for (; i < p1 && arrive_round[i] == g; i++) {
                        for (; k < l1; k++)
                            if (releases[k].round == g) {
                                if (releases[k].clock > now[i]) break;
                                rel_iround[k] = (int32_t)rd_ext.size() - e0;
                            }
                        rd_clock.push_back(now[i]);
                        rd_pods.insert(rd_pods.end(), {c0 + i - p0, c0 + i - p0 + 1});
                        rd_ext.push_back(g);
                    }
                    for (; k < l1; k++)
                        if (releases[k].round == g) rel_iround[k] = (int32_t)rd_ext.size() - e0;
                    rd_clock.push_back(round_clock[round_start[s] + g - 1]);
                    rd_pods.insert(rd_pods.end(), {c0, c0 + i - p0});
                    rd_ext.push_back(g);
                }
            } else if (round_start) {
                rd_clock.insert(rd_clock.end(), round_clock + round_start[s], round_clock + round_start[s + 1]);
            }
            rd_off.push_back((int32_t)rd_clock.size());
            sl_start.push_back((int32_t)n_slots);
            touches = std::min(n_s * (1 + R_s) + (with_releases ? rel_nodes[s] : 0), (int64_t)h->n_nodes);
        }
        if (with_releases) {
            const int t0 = track_start ? track_start[s] : 0, t1 = track_start ? track_start[s + 1] : 0;
            const int row0 = (int)tr_node.size() - t0;                /* call-wide row -> compacted row */
            for (int t = t0; t < t1; t++) {
                tr_node.push_back(tracked[t]);
                for (int i = 0; i < NHD_MAX_NICS; i++) tr_count.push_back(pods_used[(size_t)t * NHD_MAX_NICS + i]);
            }
            tr_off.push_back((int32_t)tr_node.size());
            for (int k = rel_start ? rel_start[s] : 0; k < (rel_start ? rel_start[s + 1] : 0); k++) {
                rl_rec.push_back(releases[k]);
                if (arrivals) rl_rec.back().round = rel_iround[k];      /* the kernel's round it precedes */
                rl_row.push_back(row0 + rel_row[k]);
            }
            rl_off.push_back((int32_t)rl_rec.size());
        }
        n_slots += (size_t)(touches + (edit_start ? edit_start[s + 1] - edit_start[s] : 0) +
                            (add_start ? add_start[s + 1] - add_start[s] : 0));
    }
    if (n_slots > (size_t)INT32_MAX) return fail(h, NHD_ERR_INVALID, "%zu working slots exceed the int32 range", n_slots);
    const int n_acc = (int)acc.size(), n_run = pod_off.back(), n_ed = ed_off.back(), n_ad = ad_off.back();
    if (n_run == 0) return NHD_OK;
    const bool compact = n_run != n_pods;
    std::vector<nhd_pod> cpods;
    std::vector<double> cnow;
    if (compact) {
        cpods.reserve(n_run);
        cnow.reserve(n_run);
        for (int s : acc) {
            cpods.insert(cpods.end(), pods + pod_start[s], pods + pod_start[s + 1]);
            cnow.insert(cnow.end(), now + pod_start[s], now + pod_start[s + 1]);
        }
    }
    Workspace& w = h->scratch;
    if ((rc = stage_pods(h, w, n_run, compact ? cpods.data() : pods, compact ? cnow.data() : now, max_numa)) != NHD_OK)
        return rc;

    std::vector<int32_t> idx;
    idx.reserve(pod_off.size() + ex_off.size() + ex.size() + ed_off.size() + ed_node.size() + lift.size() +
                ad_off.size() + ad_at.size() + rd_off.size() + sl_start.size() + tr_off.size() + tr_node.size() +
                rl_off.size() + rl_row.size() + rd_pods.size());
    for (const auto* v : {&pod_off, &ex_off, &ex, &ed_off, &ed_node, &lift, &ad_off, &ad_at, &rd_off, &sl_start, &tr_off,
                          &tr_node, &rl_off, &rl_row, &rd_pods})
        idx.insert(idx.end(), v->begin(), v->end());
    const size_t off_ex_off = pod_off.size(), off_ex = off_ex_off + ex_off.size(), off_ed_off = off_ex + ex.size();
    const size_t off_ed_node = off_ed_off + ed_off.size(), off_lift = off_ed_node + ed_node.size();
    const size_t off_ad_off = off_lift + lift.size(), off_ad_at = off_ad_off + ad_off.size();
    const size_t off_rd_off = off_ad_at + ad_at.size(), off_sl = off_rd_off + rd_off.size();
    const size_t off_tr_off = off_sl + sl_start.size(), off_tr_node = off_tr_off + tr_off.size();
    const size_t off_rl_off = off_tr_node + tr_node.size(), off_rl_row = off_rl_off + rl_off.size();
    const size_t off_rd_pods = off_rl_row + rl_row.size();
    const size_t off_nodes = idx.size(), off_bad = off_nodes + n_slots, off_round = off_bad + 1;
    const size_t off_count = off_round + (rounds ? n_run : 0);     /* with releases: the tracked counts */
    /* d_swork: the working slots, then the edit records and the added records the kernel seeds them from, then (with
     * rounds) the round clocks and the clocks of each pod's last attempt (reasons' base pass), 16-byte chunks */
    const size_t rd_chunks = rounds ? (rd_clock.size() + 1) / 2 : 0, last_chunks = rounds && why_counts ? ((size_t)n_run + 1) / 2 : 0;
    CK(h->d_sidx.grow((off_count + tr_count.size()) * 4));
    CK(h->d_swork.grow((n_slots + n_ed + n_ad) * sizeof(nhd_node_rec) + (rd_chunks + last_chunks) * 16));
    CK(cudaMemcpyAsync(h->d_sidx, idx.data(), idx.size() * 4, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemsetAsync(h->d_sidx + off_bad, 0, 4, h->stream));
    uint4* d_edit_rec = h->d_swork + n_slots * REC_CHUNKS;
    uint4* d_add_rec = d_edit_rec + (size_t)n_ed * REC_CHUNKS;
    double* d_round_clock = reinterpret_cast<double*>(d_add_rec + (size_t)n_ad * REC_CHUNKS);
    double* d_last_now = d_round_clock + 2 * rd_chunks;
    if (n_ed > 0)
        CK(cudaMemcpyAsync(d_edit_rec, ed_rec.data(), (size_t)n_ed * sizeof(nhd_node_rec), cudaMemcpyHostToDevice, h->stream));
    if (n_ad > 0)
        CK(cudaMemcpyAsync(d_add_rec, ad_rec.data(), (size_t)n_ad * sizeof(nhd_node_rec), cudaMemcpyHostToDevice, h->stream));
    if (!rd_clock.empty())
        CK(cudaMemcpyAsync(d_round_clock, rd_clock.data(), rd_clock.size() * 8, cudaMemcpyHostToDevice, h->stream));
    if (!tr_count.empty())
        CK(cudaMemcpyAsync(h->d_sidx + off_count, tr_count.data(), tr_count.size() * 4, cudaMemcpyHostToDevice, h->stream));
    if (!rl_rec.empty()) {  /* the accepted scenarios' releases, in place of the call's that the check read */
        CK(h->d_rels.grow(rl_rec.size() * sizeof(nhd_release)));
        CK(cudaMemcpyAsync(h->d_rels, rl_rec.data(), rl_rec.size() * sizeof(nhd_release), cudaMemcpyHostToDevice, h->stream));
    }
    if (why_counts) {       /* scenario_reasons' buffers: base rows | rows, base_row | keys | corrections, node lists */
        CK(h->d_xcounts.grow((size_t)2 * n_run * NHD_WHY_COUNT * 4));
        CK(h->d_xpod.grow((size_t)n_run * (NHD_WHY_COUNT + 3) * 4));
        CK(h->d_xnode.grow(((size_t)2 * h->n_nodes + 1) * 4));
        CK(h->d_xsmall.grow(16));
    }

    /* the candidate bitmaps of the call's pod types on the unchanged source records */
    if ((rc = launch_solve(h, w, records, false, false, true)) != NHD_OK) return rc;

    ScenarioArgs sa;
    sa.nodes = records; sa.types = w.types; sa.pod_type = w.pod_type(); sa.now = w.now();
    sa.bitmaps = w.bitmaps; sa.pod_groups = w.pod_groups(); sa.names_used = w.names_used;
    sa.pod_start = h->d_sidx; sa.excl_start = h->d_sidx + off_ex_off; sa.excl = h->d_sidx + off_ex;
    sa.lift = h->d_sidx + off_lift; sa.edit_start = h->d_sidx + off_ed_off; sa.edit_node = h->d_sidx + off_ed_node;
    sa.edit_rec = d_edit_rec;
    sa.add_start = h->d_sidx + off_ad_off; sa.add_at = h->d_sidx + off_ad_at; sa.add_rec = d_add_rec;
    sa.work = h->d_swork; sa.work_node = h->d_sidx + off_nodes; sa.out = w.out; sa.bad = (uint32_t*)(h->d_sidx + off_bad);
    sa.n_scenarios = n_acc; sa.n_types = w.n_types; sa.words = h->words; sa.n_nodes = h->n_nodes;
    sa.min_busy = h->params.min_busy_secs;
    memcpy(sa.cap, h->cap, sizeof(sa.cap));
    sa.why_delta = why_counts ? h->d_xpod + 2 * (size_t)n_run : nullptr;
    sa.round_start = h->d_sidx + off_rd_off; sa.round_clock = d_round_clock; sa.slot_start = h->d_sidx + off_sl;
    sa.pod_round = h->d_sidx + off_round;
    sa.track_start = h->d_sidx + off_tr_off; sa.tracked = h->d_sidx + off_tr_node; sa.count = h->d_sidx + off_count;
    sa.rel_start = h->d_sidx + off_rl_off; sa.rel = h->d_rels; sa.rel_track = h->d_sidx + off_rl_row;
    sa.round_pods = h->d_sidx + off_rd_pods;
    if (arrivals)           /* not NHD_PLACED until attempted: an arrival's first round walks it, releases see it */
        CK(cudaMemsetAsync(w.out, 0xFF, (size_t)n_run * sizeof(nhd_binding), h->stream));
    const int warps_per_cta = SCENARIO_THREADS / 32;
    const int grid = std::min((n_acc + warps_per_cta - 1) / warps_per_cta, h->sm_count * 16);
    /* through a pointer: the CPU emulation (tests/emu) rewrites a launch into a macro call, whose argument list would
     * split a kernel name with two template arguments */
    void (*const kernel)(ScenarioArgs) =
        arrivals      ? (why_counts ? scenario_plan_kernel<true, true, true, true> : scenario_plan_kernel<false, true, true, true>)
        : with_releases ? (why_counts ? scenario_plan_kernel<true, true, true> : scenario_plan_kernel<false, true, true>)
        : rounds      ? (why_counts ? scenario_plan_kernel<true, true> : scenario_plan_kernel<false, true>)
                      : (why_counts ? scenario_plan_kernel<true, false> : scenario_plan_kernel<false, false>);
    kernel<<<grid, SCENARIO_THREADS, 0, h->stream>>>(sa);
    CK(cudaGetLastError());
    uint32_t bad = 0;
    CK(cudaMemcpyAsync(&bad, h->d_sidx + off_bad, 4, cudaMemcpyDeviceToHost, h->stream));
    std::vector<int32_t> run_round;
    if (rounds) {
        run_round.resize(n_run);
        CK(cudaMemcpyAsync(run_round.data(), h->d_sidx + off_round, (size_t)n_run * 4, cudaMemcpyDeviceToHost, h->stream));
    }
    std::vector<nhd_binding> run;
    if (compact) run.resize(n_run);
    if ((rc = fetch_bindings(h, w, n_run, compact ? run.data() : out)) != NHD_OK) return rc;
    if (bad) return fail(h, NHD_ERR_STATE, "%s: %u chosen nodes without a mapping", what, bad);
    std::vector<uint32_t> run_rows;
    const double* run_now = compact ? cnow.data() : now;
    std::vector<double> last_now;
    if (rounds && (why_counts || pod_clock)) {  /* the clock of each pod's last attempt (its kernel round's) */
        last_now.resize(n_run);
        for (int k = 0; k < n_acc; k++)
            for (int i = pod_off[k]; i < pod_off[k + 1]; i++)
                last_now[i] = run_round[i] == 0 ? run_now[i] : rd_clock[rd_off[k] + run_round[i] - 1];
    }
    if (why_counts) {
        if (compact) run_rows.resize((size_t)n_run * NHD_WHY_COUNT);
        if (rounds) {            /* the base pass evaluates each pod at the clock of its last attempt */
            CK(cudaMemcpyAsync(d_last_now, last_now.data(), (size_t)n_run * 8, cudaMemcpyHostToDevice, h->stream));
            run_now = last_now.data();
        }
        if ((rc = scenario_reasons(h, w, records, n_run, compact ? cpods.data() : pods, run_now,
                                   rounds ? d_last_now : nullptr, compact ? run.data() : out,
                                   compact ? run_rows.data() : why_counts, what)) != NHD_OK)
            return rc;
    }
    if (arrivals)                /* kernel rounds -> the call's rounds: an arrival or a scan of gap g reads g */
        for (int k = 0; k < n_acc; k++)
            for (int i = pod_off[k]; i < pod_off[k + 1]; i++) run_round[i] = rd_ext[rd_off[k] + k + run_round[i]];
    if (rounds && !compact && pod_round) memcpy(pod_round, run_round.data(), (size_t)n_run * 4);
    if (pod_clock)
        for (int k = 0; k < n_acc; k++)
            for (int i = pod_off[k]; i < pod_off[k + 1]; i++)
                pod_clock[pod_start[acc[k]] + i - pod_off[k]] = rounds ? last_now[i] : run_now[i];
    if (compact)
        for (int k = 0; k < n_acc; k++) {
            const size_t n_k = (size_t)(pod_off[k + 1] - pod_off[k]);
            nhd_binding* o = out + pod_start[acc[k]];
            memcpy(o, run.data() + pod_off[k], n_k * sizeof(nhd_binding));
            if (n_ad > 0)                          /* added nodes by their call-wide index, as the caller numbered them */
                for (size_t i = 0; i < n_k; i++)
                    if (o[i].node >= h->n_nodes) o[i].node += add_start[acc[k]] - ad_off[k];
            if (why_counts)
                memcpy(why_counts + (size_t)pod_start[acc[k]] * NHD_WHY_COUNT,
                       run_rows.data() + (size_t)pod_off[k] * NHD_WHY_COUNT, n_k * NHD_WHY_COUNT * 4);
            if (rounds && pod_round) memcpy(pod_round + pod_start[acc[k]], run_round.data() + pod_off[k], n_k * 4);
        }
    return NHD_OK;
}

extern "C" int32_t nhd_plan_scenarios(nhd_handle* h, int32_t source, int32_t n_scenarios, const int32_t* excl_start,
                                      const int32_t* excluded, const int32_t* pod_start, const nhd_pod* pods,
                                      const double* now, nhd_binding* out, int32_t* scenario_status,
                                      int32_t* scenario_pod)
{
    return plan_scenarios(h, "nhd_plan_scenarios", source, n_scenarios, excl_start, excluded, nullptr, nullptr, nullptr,
                          nullptr, nullptr, nullptr, nullptr, pod_start, pods, now, nullptr, nullptr, nullptr,
                          nullptr, nullptr, nullptr, nullptr, out, scenario_status, scenario_pod, nullptr, nullptr);
}

extern "C" int32_t nhd_plan_scenarios_edited(nhd_handle* h, int32_t source, int32_t n_scenarios,
                                             const int32_t* excl_start, const int32_t* excluded, const int32_t* lift_at,
                                             const int32_t* edit_start, const int32_t* edit_node,
                                             const nhd_node_rec* edit_rec, const int32_t* pod_start, const nhd_pod* pods,
                                             const double* now, nhd_binding* out, int32_t* scenario_status,
                                             int32_t* scenario_pod)
{
    return plan_scenarios(h, "nhd_plan_scenarios_edited", source, n_scenarios, excl_start, excluded, lift_at,
                          edit_start, edit_node, edit_rec, nullptr, nullptr, nullptr, pod_start, pods, now, nullptr,
                          nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, out, scenario_status, scenario_pod, nullptr,
                          nullptr);
}

extern "C" int32_t nhd_plan_scenarios_explained(nhd_handle* h, int32_t source, int32_t n_scenarios,
                                                const int32_t* excl_start, const int32_t* excluded,
                                                const int32_t* lift_at, const int32_t* edit_start,
                                                const int32_t* edit_node, const nhd_node_rec* edit_rec,
                                                const int32_t* pod_start, const nhd_pod* pods, const double* now,
                                                nhd_binding* out, int32_t* scenario_status, int32_t* scenario_pod,
                                                uint32_t* why_counts)
{
    return plan_scenarios(h, "nhd_plan_scenarios_explained", source, n_scenarios, excl_start, excluded, lift_at,
                          edit_start, edit_node, edit_rec, nullptr, nullptr, nullptr, pod_start, pods, now, nullptr,
                          nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, out, scenario_status, scenario_pod,
                          why_counts, nullptr);
}

extern "C" int32_t nhd_plan_scenarios_grown(nhd_handle* h, int32_t source, int32_t n_scenarios,
                                            const int32_t* excl_start, const int32_t* excluded, const int32_t* lift_at,
                                            const int32_t* edit_start, const int32_t* edit_node,
                                            const nhd_node_rec* edit_rec, const int32_t* add_start,
                                            const int32_t* add_at, const nhd_node_rec* add_rec,
                                            const int32_t* pod_start, const nhd_pod* pods, const double* now,
                                            nhd_binding* out, int32_t* scenario_status, int32_t* scenario_pod,
                                            uint32_t* why_counts)
{
    return plan_scenarios(h, "nhd_plan_scenarios_grown", source, n_scenarios, excl_start, excluded, lift_at,
                          edit_start, edit_node, edit_rec, add_start, add_at, add_rec, pod_start, pods, now, nullptr,
                          nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, out, scenario_status, scenario_pod,
                          why_counts, nullptr);
}

extern "C" int32_t nhd_plan_scenarios_rounds(nhd_handle* h, int32_t source, int32_t n_scenarios,
                                             const int32_t* excl_start, const int32_t* excluded, const int32_t* lift_at,
                                             const int32_t* edit_start, const int32_t* edit_node,
                                             const nhd_node_rec* edit_rec, const int32_t* add_start,
                                             const int32_t* add_at, const nhd_node_rec* add_rec,
                                             const int32_t* pod_start, const nhd_pod* pods, const double* now,
                                             const int32_t* round_start, const double* round_clock, nhd_binding* out,
                                             int32_t* scenario_status, int32_t* scenario_pod, uint32_t* why_counts,
                                             int32_t* pod_round)
{
    return plan_scenarios(h, "nhd_plan_scenarios_rounds", source, n_scenarios, excl_start, excluded, lift_at,
                          edit_start, edit_node, edit_rec, add_start, add_at, add_rec, pod_start, pods, now,
                          round_start, round_clock, nullptr, nullptr, nullptr, nullptr, nullptr, out, scenario_status,
                          scenario_pod, why_counts, pod_round);
}

extern "C" int32_t nhd_plan_scenarios_releases(nhd_handle* h, int32_t source, int32_t n_scenarios,
                                               const int32_t* excl_start, const int32_t* excluded, const int32_t* lift_at,
                                               const int32_t* edit_start, const int32_t* edit_node,
                                               const nhd_node_rec* edit_rec, const int32_t* add_start,
                                               const int32_t* add_at, const nhd_node_rec* add_rec,
                                               const int32_t* pod_start, const nhd_pod* pods, const double* now,
                                               const int32_t* round_start, const double* round_clock,
                                               const int32_t* track_start, const int32_t* tracked,
                                               const int16_t* pods_used, const int32_t* rel_start,
                                               const nhd_release* releases, nhd_binding* out, int32_t* scenario_status,
                                               int32_t* scenario_pod, uint32_t* why_counts, int32_t* pod_round)
{
    return plan_scenarios(h, "nhd_plan_scenarios_releases", source, n_scenarios, excl_start, excluded, lift_at,
                          edit_start, edit_node, edit_rec, add_start, add_at, add_rec, pod_start, pods, now,
                          round_start, round_clock, track_start, tracked, pods_used, rel_start, releases, out,
                          scenario_status, scenario_pod, why_counts, pod_round);
}

extern "C" int32_t nhd_plan_scenarios_arrivals(nhd_handle* h, int32_t source, int32_t n_scenarios,
                                               const int32_t* excl_start, const int32_t* excluded, const int32_t* lift_at,
                                               const int32_t* edit_start, const int32_t* edit_node,
                                               const nhd_node_rec* edit_rec, const int32_t* add_start,
                                               const int32_t* add_at, const nhd_node_rec* add_rec,
                                               const int32_t* pod_start, const nhd_pod* pods, const double* now,
                                               const int32_t* round_start, const double* round_clock,
                                               const int32_t* track_start, const int32_t* tracked,
                                               const int16_t* pods_used, const int32_t* rel_start,
                                               const nhd_release* releases, const int32_t* arrive_round,
                                               nhd_binding* out, int32_t* scenario_status, int32_t* scenario_pod,
                                               uint32_t* why_counts, int32_t* pod_round, double* pod_clock)
{
    return plan_scenarios(h, "nhd_plan_scenarios_arrivals", source, n_scenarios, excl_start, excluded, lift_at,
                          edit_start, edit_node, edit_rec, add_start, add_at, add_rec, pod_start, pods, now,
                          round_start, round_clock, track_start, tracked, pods_used, rel_start, releases, out,
                          scenario_status, scenario_pod, why_counts, pod_round, arrive_round, pod_clock);
}

/* debug: 16 cycle accumulators + 16 counters of the last sweep (only filled by NHD_PROFILE builds) */
extern "C" int32_t nhd_debug_counters(nhd_handle* h, uint64_t* out32)
{
    if (!h || !out32) return NHD_ERR_INVALID;
#ifdef NHD_CHECKS
    cudaStreamSynchronize(h->stream);
    memcpy(out32, h->d_prof, 64 * 8);
    memset(h->d_prof, 0, 64 * 8);
    return NHD_OK;
#endif
    CK(cudaSetDevice(h->params.device));
    CK(cudaStreamSynchronize(h->stream));
    CK(cudaMemcpy(out32, h->batch.prof, 64 * 8, cudaMemcpyDeviceToHost));
    CK(cudaMemset(h->batch.prof, 0, 64 * 8));
    return NHD_OK;
}

/* Page-locked host memory for records / pods / bindings: buffers from here are copied to and
 * from the device without an intermediate staging copy. */
extern "C" int32_t nhd_alloc_pinned(uint64_t bytes, void** out)
{
    if (!out) return NHD_ERR_INVALID;
    *out = nullptr;
    return cudaMallocHost(out, bytes ? bytes : 1) == cudaSuccess ? NHD_OK : NHD_ERR_CUDA;
}

extern "C" int32_t nhd_free_pinned(void* p)
{
    if (!p) return NHD_OK;
    return cudaFreeHost(p) == cudaSuccess ? NHD_OK : NHD_ERR_CUDA;
}
