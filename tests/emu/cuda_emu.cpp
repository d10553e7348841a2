/* cuda_emu.cpp — TEST INFRASTRUCTURE: fiber scheduler behind tests/emu/cuda_emu.h. */
#include "cuda_emu.h"

#include <stdarg.h>

dim3 threadIdx, blockIdx, blockDim, gridDim;

/* marks a library built on this emulation: nhd_b200/_lib.py refuses to load one unless the caller says so */
extern "C" int nhd_emulated_device() { return 1; }

namespace emu {

Block* g_blk = nullptr;
const char* g_kernel_name = "?";
size_t g_stack_bytes = 512 * 1024;
static Block g_block;

[[noreturn]] void fail(const char* fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    fprintf(stderr, "cuda_emu: kernel %s, block %u, thread %u: ", g_kernel_name, blockIdx.x, threadIdx.x);
    vfprintf(stderr, fmt, ap);
    fprintf(stderr, "\n");
    va_end(ap);
    fflush(stderr);
    abort();
}

void yield()
{
    Block* b = g_blk;
    swapcontext(&b->fibers[b->cur].ctx, &b->sched);
}

static const char* op_name(int op)
{
    switch (op) { case OP_SHFL: return "__shfl_sync"; case OP_SHFL_UP: return "__shfl_up_sync"; case OP_BALLOT: return "__ballot_sync";
                  case OP_ALL: return "__all_sync"; case OP_SYNCWARP: return "__syncwarp"; default: return "?"; }
}

uint64_t collective(int op, uint32_t mask, uint64_t val, int arg, int line)
{
    Block* b = g_blk;
    const unsigned tid = b->fibers[b->cur].tid, lane = tid & 31, wid = tid >> 5;
    Warp& w = b->warps[wid];
    { Fiber& me = b->fibers[b->cur]; me.hist[me.nhist++ % 12] = line; }
    const unsigned lanes_here = (b->n - wid * 32) >= 32 ? 32u : (unsigned)(b->n - wid * 32);
    const uint32_t exist = lanes_here == 32 ? 0xFFFFFFFFu : ((1u << lanes_here) - 1);
    if (!(mask & (1u << lane))) fail("%s: the calling lane %u is not in its own mask %08x", op_name(op), lane, mask);
    if (mask == 0xFFFFFFFFu && exist != 0xFFFFFFFFu) mask = exist;      /* partial last warp */
    if (mask & ~exist) fail("%s: mask %08x names lanes that do not exist", op_name(op), mask);
    for (unsigned j = 0; j < 32; j++) {
        if (!((mask >> j) & 1) || j == lane) continue;
        if (b->fibers[wid * 32 + j].state == ST_DONE)
            fail("%s with mask %08x: lane %u has already left the kernel", op_name(op), mask, j);
        if ((w.waiting >> j) & 1) {
            if (w.slot[j].mask != mask || w.slot[j].op != op) {
                for (unsigned who : {lane, j}) {
                    Fiber& f = b->fibers[wid * 32 + who];
                    fprintf(stderr, "cuda_emu: lane %u came through lines", who);
                    for (unsigned k = f.nhist > 12 ? f.nhist - 12 : 0; k < f.nhist; k++) fprintf(stderr, " %d", f.hist[k % 12]);
                    fprintf(stderr, "\n");
                }
                fail("divergent collectives in warp %u: lane %u is in %s(mask %08x) at line %d, lane %u in %s(mask %08x) at line %d",
                     wid, lane, op_name(op), mask, line, j, op_name(w.slot[j].op), w.slot[j].mask, w.slot[j].line);
            }
        }
    }
    w.slot[lane].op = op; w.slot[lane].mask = mask; w.slot[lane].val = val; w.slot[lane].arg = arg; w.slot[lane].line = line;
    w.waiting |= 1u << lane;
    if ((w.waiting & mask) == mask) {                       /* last to arrive: work out everybody's result */
        uint64_t ballot = 0; int all = 1;
        for (unsigned j = 0; j < 32; j++) if ((mask >> j) & 1) { if (w.slot[j].val & 1) ballot |= 1ull << j; else all = 0; }
        for (unsigned j = 0; j < 32; j++) {
            if (!((mask >> j) & 1)) continue;
            switch (op) {
            case OP_SHFL: { const unsigned src = (unsigned)w.slot[j].arg & 31;
                            w.result[j] = ((mask >> src) & 1) ? w.slot[src].val : w.slot[j].val; break; }
            case OP_SHFL_UP: { const int src = (int)j - w.slot[j].arg;
                               w.result[j] = (src >= 0 && ((mask >> src) & 1)) ? w.slot[src].val : w.slot[j].val; break; }
            case OP_BALLOT: w.result[j] = ballot; break;
            case OP_ALL: w.result[j] = (uint64_t)all; break;
            default: w.result[j] = 0;
            }
        }
        w.waiting &= ~mask;
        w.released |= mask;
        for (unsigned j = 0; j < 32; j++) if ((mask >> j) & 1) b->fibers[wid * 32 + j].state = ST_RUN;
        b->progress++;
        b->completed_warp = (int)wid;
        yield();                                   /* the lanes resume in scheduler order, not "last arriver first" */
    }
    while (!((w.released >> lane) & 1)) {
        b->fibers[b->cur].state = ST_COLL;
        yield();
    }
    w.released &= ~(1u << lane);
    return w.result[lane];
}

void syncthreads()
{
    Block* b = g_blk;
    const unsigned gen = b->sync_gen;
    b->sync_waiting++;
    if (b->sync_waiting == b->live) {
        b->sync_waiting = 0; b->sync_gen++; b->progress++;
        for (auto& f : b->fibers) if (f.state == ST_SYNC) f.state = ST_RUN;
        return;
    }
    while (b->sync_gen == gen) {
        b->fibers[b->cur].state = ST_SYNC;
        yield();
    }
}

static void trampoline()
{
    Block* b = g_blk;
    b->body();
    Fiber& f = b->fibers[b->cur];
    f.state = ST_DONE;
    b->live--;
    b->progress++;
    if (b->sync_waiting > 0 && b->sync_waiting == b->live) {     /* an exited thread no longer holds a barrier up */
        b->sync_waiting = 0; b->sync_gen++;
        for (auto& g : b->fibers) if (g.state == ST_SYNC) g.state = ST_RUN;
    }
    swapcontext(&f.ctx, &b->sched);
    abort();
}

}  // namespace emu

namespace nhd { alignas(1024) uint8_t smem[256 * 1024]; }     /* `extern __shared__ uint8_t smem[]` of the kernels */

namespace emu {

void run_grid(const char* name, dim3 grid, dim3 block, size_t dyn_smem, std::function<void()> body)
{
    if (g_blk) fail("nested kernel launch");
    if ((block.x * block.y * block.z + 31) / 32 > 64) fail("blocks of more than 64 warps are not supported");
    if (dyn_smem > 227 * 1024 || dyn_smem > sizeof(nhd::smem))          /* sharedMemPerBlockOptin of the emulated device */
        fail("launch asks for %zu bytes of dynamic shared memory (the H100 allows 232448)", dyn_smem);
    if (block.x * block.y * block.z > 1024) fail("launch with %u threads per block", block.x * block.y * block.z);
    Block& b = g_block;
    const int n = (int)(block.x * block.y * block.z);
    g_kernel_name = name;
    gridDim = grid; blockDim = block;
    if ((size_t)n * g_stack_bytes > b.stacks.size()) b.stacks.resize((size_t)n * g_stack_bytes);
    b.body = body;
    for (unsigned bz = 0; bz < grid.z; bz++) for (unsigned by = 0; by < grid.y; by++) for (unsigned bx = 0; bx < grid.x; bx++) {
        blockIdx = dim3(bx, by, bz);
        memset(nhd::smem, 0xCD, dyn_smem);                       /* shared memory is NOT zero on entry */
        b.fibers.assign(n, Fiber());
        b.warps.assign((n + 31) / 32, Warp());
        for (auto& w : b.warps) { w.waiting = 0; w.released = 0; }
        b.n = n; b.live = n; b.sync_waiting = 0; b.sync_gen = 0;
        g_blk = &b;
        for (int t = 0; t < n; t++) {
            Fiber& f = b.fibers[t];
            f.state = ST_RUN; f.tid = (unsigned)t; f.nhist = 0;
            getcontext(&f.ctx);
            f.ctx.uc_stack.ss_sp = b.stacks.data() + (size_t)t * g_stack_bytes;
            f.ctx.uc_stack.ss_size = g_stack_bytes;
            f.ctx.uc_link = nullptr;
            makecontext(&f.ctx, trampoline, 0);
        }
        unsigned long long idle_rounds = 0, last_progress = b.progress;
        static const bool descending = getenv("EMU_LANE_ORDER") && getenv("EMU_LANE_ORDER")[0] == 'd';
        while (b.live > 0) {
            bool ran = false;
            /* warps take turns; inside a warp the lanes run in a fixed order (ascending, or descending with
             * EMU_LANE_ORDER=d), and whenever one of the warp's collectives completes the order starts over, so
             * that between two collectives the lanes of a warp always execute in that order — the closest a
             * run-to-the-next-collective emulation gets to a converged warp (see README in cuda_emu.h) */
            const int n_warps = (n + 31) / 32;
            /* EMU_SCHED_SEED=<n>: the warps are visited in a pseudo-random order that changes every round, and a
             * warp may be skipped for a round — other interleavings of the inter-warp protocols (turn counters,
             * caches shared by several warps) than plain round-robin */
            static const char* seed_env = getenv("EMU_SCHED_SEED");
            static uint64_t rng = seed_env ? 0x9E3779B97F4A7C15ull * (uint64_t)(atoll(seed_env) + 1) : 0;
            int order[64];
            for (int i = 0; i < n_warps && i < 64; i++) order[i] = descending ? n_warps - 1 - i : i;
            if (seed_env)
                for (int i = n_warps - 1; i > 0; i--) {
                    rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;
                    const int j = (int)(rng % (uint64_t)(i + 1));
                    const int tmp = order[i]; order[i] = order[j]; order[j] = tmp;
                }
            for (int wk = 0; wk < n_warps && b.live > 0; wk++) {
                const int wi = order[wk];
                if (seed_env) { rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17; if ((rng & 3) == 0) { ran = true; continue; } }
                const int lanes = (n - wi * 32) >= 32 ? 32 : n - wi * 32;
                int restarts = 0;
                for (int k = 0; k < lanes && b.live > 0; k++) {
                    const int t = wi * 32 + (descending ? lanes - 1 - k : k);
                    Fiber& f = b.fibers[t];
                    if (f.state != ST_RUN) continue;
                    ran = true;
                    b.cur = t;
                    threadIdx = dim3((unsigned)t % block.x, ((unsigned)t / block.x) % block.y, (unsigned)t / (block.x * block.y));
                    b.completed_warp = -1;
                    swapcontext(&b.sched, &f.ctx);
                    if (b.completed_warp == wi && restarts < 64) { restarts++; k = -1; }
                }
            }
            if (!ran && b.live > 0) {
                int coll = 0, sync = 0;
                for (auto& f : b.fibers) { coll += f.state == ST_COLL; sync += f.state == ST_SYNC; }
                b.cur = 0; threadIdx = dim3(0, 0, 0);
                fail("deadlock: %d threads wait in a warp collective, %d at __syncthreads, nobody can run", coll, sync);
            }
            if (b.progress == last_progress) {
                if (++idle_rounds > 2000000ull) { b.cur = 0; fail("no progress for 2e6 scheduler rounds (spin loop that never ends?)"); }
            } else { idle_rounds = 0; last_progress = b.progress; }
        }
        g_blk = nullptr;
    }
}

}  // namespace emu
