// bioik_capi.cu — host side of libbioik_b200.so: the C ABI of include/bioik_b200.h.
// Flattens the robot/problem tables (the host-side halves of IKBase::initialize /
// RobotFK_Fast_Base::initialize / RobotFK_Jacobian::initialize), generates the reference's
// RNG lookup tables, owns device memory and the stream, and launches the kernels of
// bioik_kernels.cuh.  No CPU compute path exists here: every solve runs on the GPU.
#include "../../include/bioik_b200.h"
#include "bioik_host.hpp"
#include "bioik_kernels.cuh"

#include <cuda_runtime.h>
#include <pthread.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <random>
#include <cstdio>
#include <string>
#include <vector>

using namespace bioik;

namespace
{
thread_local std::string g_create_error;

struct EventPair
{
    cudaEvent_t a, b;
    int kind; // 0 = evolve, 1 = serial
};
} // namespace

// launch plan and progress of the solve in flight (bioik_begin .. bioik_get_solution, or one bioik_solve_* call)
struct RunPlan
{
    bool open = false;     // solve_begin has run
    bool prepared = false; // the approximator (tip frames, delta frames) of step next_step is in the state
    int B = 0, next_step = 0;
    int Q = 0, islands = 0; // bioik_begin: queries x islands (0: plain batch)
    EvolveFastKernel fast = nullptr;
    int evolve_lpt = 32; // lanes per task of the generation kernel
    int evolve_wpb = BIOIK_EVOLVE_WPB; // warps per block of the generation kernel
    size_t evolve_smem = 0;
    MemeticGroupKernel mgk = nullptr;
    int mg_width = 8, mg_warps = 4;
    size_t mg_smem = 0;
    bool use_mg = false, stale = false;
    const char* dominant = ""; // instantiation name of the kernel bioik_kernel_time times as "generation" work
    PersistKernel persist = nullptr; // one launch for many steps (bioik_persist.cuh); nullptr: one launch per step and kernel
    size_t persist_smem = 0;
    int persist_blocks_per_sm = 0;
};

struct bioik_ctx
{
    BioikSolverCfg cfg;
    HostRobot robot;
    cudaStream_t stream = nullptr;
    int serial_plan_force = -1;
    int lpt_want = 16; // BIOIK_EVOLVE_LPT: lanes per task of the single-pose generation kernel (8, 16 or 32; 16 was the fastest on cfg2)
    int ch_cap = 8; // BIOIK_EVOLVE_CH: cap of the register block of k_evolve_fast (experiments)
    std::string error;
    int64_t launches = 0;
    RunPlan run;

    bool has_problem = false;
    DProblem hP;
    DProblem* dP = nullptr;

    double *d_uniform = nullptr, *d_gauss = nullptr;
    double gauss_absmax = 0; // max |gauss| of the lookup table

    // schedules (depend on steps, gens, C, n)
    int sched_steps = -1, sched_n = -1;
    int32_t* d_gauss_off = nullptr;
    uint8_t* d_rate_exp = nullptr;
    double* d_mtab = nullptr; // [calls][n][C] mutation table of the fast generation kernel
    SerialPlan splan;           // launch plan of the fused serial kernel (set_problem)
    SerialKernel serial = nullptr;
    int sm_count = 132; // H100 SXM; replaced by the device's own count when the context is created
    bool force_generic = false; // BIOIK_FORCE_GENERIC=1: always use the generic generation kernel (tests)
    bool generic_now = false;   // the solve in flight runs the generic kernels (forced, or a problem shape the fused kernels do not take)

    // state
    int capB = 0;
    DState S;
    void* state_block = nullptr;
    // staging for the host-pointer API
    int stageB = 0;
    double *d_gp = nullptr, *d_seeds = nullptr, *d_osol = nullptr, *d_ofit = nullptr;
    uint32_t* d_rs = nullptr;
    int32_t *d_osucc = nullptr, *d_osteps = nullptr;
    double* d_default_gp = nullptr; // [G][NPARAM] defaults (goal_params == NULL)

    // timing (collected only after bioik_kernel_time has been called once: events cost host time per launch)
    bool timing = false;
    bool capturing = false;
    // CUDA graph of the last host-API solve shape (B, steps, early_exit, with/without per-query goal parameters)
    cudaGraphExec_t graph_exec = nullptr;
    int graph_B = -1, graph_steps = -1, graph_early = -1, graph_gp = -1;
    int64_t graph_launches = 0;
    bool use_graphs = true; // BIOIK_NO_GRAPH=1 disables
    std::vector<EventPair> pending, pool;
    double ms_evolve = 0, ms_serial = 0;
    int64_t n_evolve = 0, n_serial = 0;
    bool stale_tips = false; // BIOIK_OPT_REFERENCE_STALE_TIPS
    int island_stride = 0;   // BIOIK_OPT_ISLAND_STREAM_STRIDE
    int memetic_group = -1; // BIOIK_MEMETIC_GROUP: 0 = memetic step inside the thread-per-task serial kernel, 1 = always k_memetic_group, unset = by problem shape
    // query-level buffers of bioik_solve_islands
    double *d_q_gp = nullptr, *d_q_seeds = nullptr, *d_q_sol = nullptr, *d_q_fit = nullptr;
    int32_t *d_q_succ = nullptr, *d_q_island = nullptr, *d_q_steps = nullptr;
    int queryQ = 0;
    int32_t* d_cancel = nullptr;          // device flag read by every kernel (run_done); set by bioik_cancel through its own stream
    int32_t* h_one = nullptr;             // pinned constant 1, the source of that copy
    cudaStream_t stream_cancel = nullptr; // so that the copy overtakes a running solve
    int32_t* d_flag = nullptr; // "any run still active" (bioik_solve_islands polls it between bursts)
    int32_t* h_flag = nullptr; // pinned host copy
    int persist_mode = 0; // BIOIK_PERSIST=1: the persistent solve kernel where it exists (bioik_persist.cuh); 0: stepped launches
    // work queues of the persistent kernel
    unsigned long long* d_queue = nullptr;
    size_t queue_slots = 0;
    int32_t *d_qctr = nullptr, *d_gcount = nullptr;
    int gcount_cap = 0;
    bool serial_split = false; // BIOIK_SERIAL_SPLIT=1: one launch per phase of the serial kernel (phase timing study)
    double ms_phase[3] = {0, 0, 0};
};

namespace
{
#define CU(ctx, call)                                                                                             \
    do                                                                                                            \
    {                                                                                                             \
        cudaError_t e_ = (call);                                                                                  \
        if(e_ != cudaSuccess)                                                                                     \
        {                                                                                                         \
            (ctx)->error = std::string(#call) + ": " + cudaGetErrorString(e_);                                    \
            return BIOIK_E_CUDA;                                                                                  \
        }                                                                                                         \
    } while(0)

int fail(bioik_ctx* ctx, int code, const std::string& msg)
{
    if(ctx)
        ctx->error = msg;
    else
        g_create_error = msg;
    return code;
}

size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

// BIOIK_TRACE=1: entry / exit of every ABI call on stderr with the calling thread (debugging of host-side integration)
struct Trace
{
    const char* name;
    bool on;
    explicit Trace(const char* n) : name(n)
    {
        static const bool enabled = getenv("BIOIK_TRACE") && getenv("BIOIK_TRACE")[0] == '1';
        on = enabled;
        if(on) fprintf(stderr, "[bioik %lx] > %s\n", (unsigned long)pthread_self(), name);
    }
    ~Trace()
    {
        if(on) fprintf(stderr, "[bioik %lx] < %s\n", (unsigned long)pthread_self(), name);
    }
};

void drop_graph(bioik_ctx* ctx);

// The three ensure_* functions may free and reallocate buffers whose addresses a cached CUDA graph of bioik_solve_batch has
// baked in: each of them drops that graph before it frees anything.
int ensure_state(bioik_ctx* ctx, int B)
{
    if(B <= ctx->capB) return BIOIK_OK;
    drop_graph(ctx);
    CU(ctx, cudaDeviceSynchronize());
    ctx->capB = 0; // a failed allocation below must not leave a stale capacity behind
    if(ctx->state_block) cudaFree(ctx->state_block);
    ctx->state_block = nullptr;
    const DProblem& P = ctx->hP;
    size_t n = P.n, T = P.T, gens = ctx->cfg.generations;
    size_t sizes[] = {
        (size_t)B * 4 * n * 8,         // genes
        (size_t)B * 4 * n * 8,         // grads
        (size_t)B * 2 * 8,             // sfit
        (size_t)B * 2 * 4,             // impr
        (size_t)B * n * 8,             // sol
        (size_t)B * 8,                 // solfit
        (size_t)B * 4,                 // rng
        (size_t)B * 4,                 // done
        (size_t)B * 4,                 // steps
        (size_t)B * 4,                 // success
        (size_t)B * 2 * gens * 4,      // ccount
        (size_t)B * 2 * n * 8,         // base
        (size_t)B * 2 * T * 7 * 8,     // tip0
        (size_t)B * 2 * T * n * 7 * 8, // delta
        (size_t)B * 4,                 // qstep
        (size_t)B * T * 7 * 8,         // carry
    };
    size_t total = 0;
    for(size_t s : sizes) total += align_up(s);
    CU(ctx, cudaMalloc(&ctx->state_block, total));
    char* p = (char*)ctx->state_block;
    auto take = [&](size_t s) {
        char* r = p;
        p += align_up(s);
        return r;
    };
    DState& S = ctx->S;
    S.genes = (double*)take(sizes[0]);
    S.grads = (double*)take(sizes[1]);
    S.sfit = (double*)take(sizes[2]);
    S.impr = (int32_t*)take(sizes[3]);
    S.sol = (double*)take(sizes[4]);
    S.solfit = (double*)take(sizes[5]);
    S.rng = (uint32_t*)take(sizes[6]);
    S.done = (int32_t*)take(sizes[7]);
    S.steps = (int32_t*)take(sizes[8]);
    S.success = (int32_t*)take(sizes[9]);
    S.ccount = (int32_t*)take(sizes[10]);
    S.base = (double*)take(sizes[11]);
    S.tip0 = (double*)take(sizes[12]);
    S.delta = (double*)take(sizes[13]);
    S.qstep = (int32_t*)take(sizes[14]);
    S.carry = (double*)take(sizes[15]);
    ctx->capB = B;
    return BIOIK_OK;
}

int ensure_staging(bioik_ctx* ctx, int B)
{
    if(B <= ctx->stageB) return BIOIK_OK;
    drop_graph(ctx);
    CU(ctx, cudaDeviceSynchronize());
    ctx->stageB = 0;
    cudaFree(ctx->d_gp), cudaFree(ctx->d_seeds), cudaFree(ctx->d_rs), cudaFree(ctx->d_osol), cudaFree(ctx->d_ofit), cudaFree(ctx->d_osucc), cudaFree(ctx->d_osteps);
    ctx->d_gp = ctx->d_seeds = ctx->d_osol = ctx->d_ofit = nullptr, ctx->d_rs = nullptr, ctx->d_osucc = ctx->d_osteps = nullptr;
    const DProblem& P = ctx->hP;
    CU(ctx, cudaMalloc(&ctx->d_gp, (size_t)B * P.G * GOAL_NPARAM * 8));
    CU(ctx, cudaMalloc(&ctx->d_seeds, (size_t)B * P.n_vars * 8));
    CU(ctx, cudaMalloc(&ctx->d_rs, (size_t)B * 4));
    CU(ctx, cudaMalloc(&ctx->d_osol, (size_t)B * P.n_vars * 8));
    CU(ctx, cudaMalloc(&ctx->d_ofit, (size_t)B * 8));
    CU(ctx, cudaMalloc(&ctx->d_osucc, (size_t)B * 4));
    CU(ctx, cudaMalloc(&ctx->d_osteps, (size_t)B * 4));
    ctx->stageB = B;
    return BIOIK_OK;
}

int check_launch(bioik_ctx* ctx, const char* what);

void drop_graph(bioik_ctx* ctx)
{
    if(ctx->graph_exec) cudaGraphExecDestroy(ctx->graph_exec), ctx->graph_exec = nullptr;
    ctx->graph_B = -1;
}

int ensure_schedules(bioik_ctx* ctx, int steps)
{
    if(ctx->sched_steps >= steps && ctx->sched_n == ctx->hP.n) return BIOIK_OK;
    if(ctx->sched_n == ctx->hP.n && ctx->sched_steps > 0) steps = std::max(steps, 2 * ctx->sched_steps); // a resumable solve grows its schedule geometrically
    std::vector<int32_t> go;
    std::vector<uint8_t> re;
    make_schedules(steps, ctx->cfg.generations, ctx->cfg.population, ctx->hP.n, go, re);
    drop_graph(ctx);
    CU(ctx, cudaDeviceSynchronize()); // kernels of a solve in flight (on any stream) may still read the old tables
    cudaFree(ctx->d_gauss_off), cudaFree(ctx->d_rate_exp), cudaFree(ctx->d_mtab);
    ctx->d_gauss_off = nullptr, ctx->d_rate_exp = nullptr, ctx->d_mtab = nullptr;
    CU(ctx, cudaMalloc(&ctx->d_gauss_off, go.size() * 4));
    CU(ctx, cudaMalloc(&ctx->d_rate_exp, re.size()));
    CU(ctx, cudaMemcpy(ctx->d_gauss_off, go.data(), go.size() * 4, cudaMemcpyHostToDevice));
    CU(ctx, cudaMemcpy(ctx->d_rate_exp, re.data(), re.size(), cudaMemcpyHostToDevice));
    {
        // query-independent mutation table of the fast generation kernel (bioik_evolve_fast.cuh)
        const int calls = (int)go.size(), C = ctx->cfg.population;
        const long long total = (long long)calls * ctx->hP.n * mtab_row(C);
        CU(ctx, cudaMalloc(&ctx->d_mtab, (size_t)total * 8));
        k_mutation_table<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>(ctx->dP, calls, C, ctx->d_gauss, ctx->d_gauss_off, ctx->d_rate_exp, ctx->d_mtab);
        int rc = check_launch(ctx, "k_mutation_table");
        if(rc != BIOIK_OK) return rc;
        CU(ctx, cudaStreamSynchronize(ctx->stream));
    }
    ctx->sched_steps = steps;
    ctx->sched_n = ctx->hP.n;
    return BIOIK_OK;
}

struct Timed // records an event pair around a launch when timing is on (and not while capturing a graph)
{
    bioik_ctx* ctx;
    cudaStream_t st;
    EventPair p;
    bool on;
    Timed(bioik_ctx* c, cudaStream_t s, int kind);
    void done();
};

EventPair get_pair(bioik_ctx* ctx, int kind)
{
    EventPair p;
    if(!ctx->pool.empty())
    {
        p = ctx->pool.back();
        ctx->pool.pop_back();
    }
    else
    {
        cudaEventCreate(&p.a);
        cudaEventCreate(&p.b);
    }
    p.kind = kind;
    return p;
}

void drain_events(bioik_ctx* ctx);

Timed::Timed(bioik_ctx* c, cudaStream_t s, int kind) : ctx(c), st(s), on(c->timing && !c->capturing)
{
    if(on)
    {
        p = get_pair(ctx, kind);
        cudaEventRecord(p.a, st);
    }
}
void Timed::done()
{
    if(on)
    {
        cudaEventRecord(p.b, st);
        ctx->pending.push_back(p);
    }
}

int check_launch(bioik_ctx* ctx, const char* what)
{
    cudaError_t e = cudaGetLastError();
    if(e != cudaSuccess)
    {
        ctx->error = std::string(what) + ": " + cudaGetErrorString(e);
        return BIOIK_E_CUDA;
    }
    ctx->launches++;
    return BIOIK_OK;
}

// [B][n_vars + 3] result slab of the multi-GPU gather: solution | fitness | success | steps (bio_ik_b200/distributed.py)
__global__ void k_pack_results(int B, int n_vars, const double* __restrict__ sol, const double* __restrict__ fit, const int32_t* __restrict__ succ, const int32_t* __restrict__ steps, double* __restrict__ slab)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int W = n_vars + 3;
    if(i >= (size_t)B * W) return;
    const int q = (int)(i / W), c = (int)(i - (size_t)q * W);
    slab[i] = c < n_vars ? sol[(size_t)q * n_vars + c] : (c == n_vars ? fit[q] : (c == n_vars + 1 ? (double)succ[q] : (double)steps[q]));
}

__global__ void k_broadcast(const double* __restrict__ src, int per, int B, double* __restrict__ dst)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(i < (size_t)B * per) dst[i] = src[i % per];
}

// ---- a solve in three parts: begin (IKBase::initialize for every run), steps [s0, s1) (IKBase::step), finish (getSolution) --------
// bioik_solve_batch* enqueue all three on one stream; bioik_begin / bioik_step / bioik_get_solution expose them one by one.

// IKEvolution2::initialize for B runs + the approximator of step 0.  All pointers are device pointers.
int solve_begin(bioik_ctx* ctx, cudaStream_t st, int B, const double* d_gp, const double* d_seeds, const uint32_t* d_rs, int total_steps, int early_exit, int islands)
{
    if(!ctx->has_problem) return fail(ctx, BIOIK_E_NO_PROBLEM, "bioik_set_problem has not been called");
    if(B <= 0 || total_steps < 0 || !d_seeds || !d_rs) return fail(ctx, BIOIK_E_INVALID, "bad solve arguments");
    int rc;
    ctx->run.open = false;
    if(ctx->pending.size() > 4096) drain_events(ctx); // bound the timing-event backlog
    if((rc = ensure_state(ctx, B)) != BIOIK_OK) return rc;
    // islands reading the random streams ahead of island 0 need that much more of the schedules
    const int stream_lead = islands > 1 ? (islands - 1) * ctx->island_stride : 0;
    if((rc = ensure_schedules(ctx, std::max(std::min(total_steps, 64), 1) + stream_lead)) != BIOIK_OK) return rc;
    const DProblem& P = ctx->hP;
    DState& S = ctx->S;
    S.B = B;
    S.C = ctx->cfg.population;
    S.gens = ctx->cfg.generations;
    S.memetic = ctx->cfg.memetic;
    S.memetic_iters = ctx->cfg.memetic_iters;
    S.total_steps = total_steps;
    S.early_exit = early_exit;
    S.islands = islands;
    S.island_stride = islands > 1 ? ctx->island_stride : 0;
    S.cancel = ctx->d_cancel;
    if(!d_gp)
    {
        // no per-query parameters: broadcast the defaults of BioikGoal::p
        if((rc = ensure_staging(ctx, B)) != BIOIK_OK) return rc;
        const int per = P.G * GOAL_NPARAM;
        k_broadcast<<<(int)(((size_t)B * per + 255) / 256), 256, 0, st>>>(ctx->d_default_gp, per, B, ctx->d_gp);
        if((rc = check_launch(ctx, "k_broadcast")) != BIOIK_OK) return rc;
        d_gp = ctx->d_gp;
    }
    S.goal_params = d_gp;
    S.seeds = d_seeds;
    S.rng_seeds = d_rs;
    S.uniform = ctx->d_uniform;
    S.gauss = ctx->d_gauss;
    S.gauss_absmax = ctx->gauss_absmax;

    // launch plan of the step kernels
    RunPlan& R = ctx->run;
    R = RunPlan();
    R.B = B;
    R.next_step = 0;
    R.evolve_lpt = 32;
    // more than 8 tips (BalanceGoal: one per link with mass): the per-task shared-memory plans of the fused kernels do not apply
    ctx->generic_now = ctx->force_generic || P.T > 8 || P.n_balance > 0;
    R.fast = ctx->generic_now ? nullptr : select_evolve_fast(P, S.C, ctx->ch_cap, &R.evolve_lpt, ctx->lpt_want);
    R.dominant = R.fast ? selected_kernel_name() : "k_evolve";
    const int warps_per_block = R.fast ? evolve_warps_per_block(R.evolve_lpt) : BIOIK_EVOLVE_WPB;
    R.evolve_wpb = warps_per_block;
    if(R.fast)
    {
        FastSmem L = fast_smem_layout(P);
        R.evolve_smem = (size_t)warps_per_block * (32 / R.evolve_lpt) * L.total() * sizeof(double);
        if(R.evolve_smem > 48 * 1024) CU(ctx, cudaFuncSetAttribute((const void*)R.fast, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)R.evolve_smem));
    }
    else
    {
        EvolveSmem L{P.n, P.T, P.G};
        R.evolve_smem = (size_t)warps_per_block * L.total() * sizeof(double);
        if(R.evolve_smem > 48 * 1024) CU(ctx, cudaFuncSetAttribute(k_evolve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)R.evolve_smem));
    }
    const int TPB = 128;
    k_init<<<(B + TPB - 1) / TPB, TPB, 0, st>>>(ctx->dP, S);
    if((rc = check_launch(ctx, "k_init")) != BIOIK_OK) return rc;
    if(!ctx->generic_now)
    {
        // production path: k_evolve_fast (or k_evolve for shapes without a fast instantiation) + the fused k_serial
        ctx->splan = make_serial_plan(P, 2 * B, ctx->sm_count);
        if(ctx->serial_plan_force >= 0)
        {
            // experiment knob BIOIK_SERIAL_PLAN: bit0 = delta frames in shared memory, bit1 = link frames in shared memory
            SerialPlan& f = ctx->splan;
            f.delta_smem = ctx->serial_plan_force & 1, f.frames_smem = (ctx->serial_plan_force >> 1) & 1;
            f.per_thread = serial_fixed_doubles(P) + (f.delta_smem ? 7 * P.T * P.n : 0) + (f.frames_smem ? 7 * P.L : 0);
            f.smem_bytes = (size_t)f.per_thread * f.block * sizeof(double);
        }
        ctx->serial = select_serial(ctx->splan);
        const SerialPlan& pl = ctx->splan;
        if(pl.smem_bytes > 48 * 1024) CU(ctx, cudaFuncSetAttribute((const void*)ctx->serial, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem_bytes));
        R.mg_width = memetic_group_width(P.n);
        // reference-quirk mode: the group kernel with one group per QUERY (the two species share the solver's phenotypes3)
        R.stale = ctx->stale_tips && S.memetic && stale_tips_matter(P);
        R.mgk = select_memetic_group(R.mg_width, R.stale);
        R.mg_warps = 4;
        const int mg_tasks_per_block = R.mg_warps * (32 / R.mg_width);
        const GroupLayout mgl{P.n, P.T, P.G, R.mg_width, P.tip_gene_start[P.T], R.stale ? 1 : 0, P.n_joint_goals};
        R.mg_smem = (size_t)mg_tasks_per_block * mgl.total() * sizeof(double);
        // the unrolled single-pose path of k_serial issues ~3x fewer instructions per task than a lane group; everything else
        // gains from the extra parallelism of the group kernel
        const bool want_mg = R.stale || (ctx->memetic_group < 0 ? !has_unrolled_memetic(P) : ctx->memetic_group != 0);
        R.use_mg = want_mg && S.memetic && R.mg_smem <= 200 * 1024;
        if(R.stale && !R.use_mg) return fail(ctx, BIOIK_E_LIMIT, "BIOIK_OPT_REFERENCE_STALE_TIPS: problem too large for the lane-group memetic kernel");
        if(R.use_mg && R.mg_smem > 48 * 1024) CU(ctx, cudaFuncSetAttribute((const void*)R.mgk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)R.mg_smem));
        // the persistent kernel: same two bodies, fed from device-side queues (one launch for many steps)
        bool pds = true, pfs = false;
        R.persist = (ctx->persist_mode && R.fast && R.evolve_lpt == 16 && !R.use_mg && !ctx->serial_split && ctx->serial_plan_force < 0) ? select_persist(P, S.C, &pds, &pfs) : nullptr;
        if(R.persist)
        {
            R.persist_smem = persist_smem_bytes(P, 16, pds, pfs);
            if(R.persist_smem > 200 * 1024)
                R.persist = nullptr;
            else
            {
                CU(ctx, cudaFuncSetAttribute((const void*)R.persist, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)R.persist_smem));
                CU(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&R.persist_blocks_per_sm, (const void*)R.persist, 32 * PERSIST_WARPS, R.persist_smem));
                if(R.persist_blocks_per_sm < 1) R.persist = nullptr;
            }
        }
        if(R.persist) R.dominant = selected_kernel_name();
    }
    else if(ctx->stale_tips && S.memetic && stale_tips_matter(P))
        return fail(ctx, BIOIK_E_LIMIT, "BIOIK_OPT_REFERENCE_STALE_TIPS is not available with BIOIK_FORCE_GENERIC");
    R.open = true;
    R.prepared = false;
    return BIOIK_OK;
}

int launch_serial(bioik_ctx* ctx, cudaStream_t st, int step, int phases)
{
    const RunPlan& R = ctx->run;
    const DState& S = ctx->S;
    const SerialPlan& pl = ctx->splan;
    const int sgrid = (2 * S.B + pl.block - 1) / pl.block;
    if(R.use_mg && (phases & PH_MEMETIC))
    {
        // the memetic line search on W lanes per task (bioik_memetic_group.cuh), then the rest of the serial work
        Timed tg(ctx, st, 2);
        const int mg_tasks_per_block = R.mg_warps * (32 / R.mg_width);
        const int mg_units = R.stale ? S.B : 2 * S.B; // groups own queries in the reference-quirk mode
        R.mgk<<<(mg_units + mg_tasks_per_block - 1) / mg_tasks_per_block, R.mg_warps * 32, R.mg_smem, st>>>(ctx->hP, S, step);
        int r = check_launch(ctx, "k_memetic_group");
        tg.done();
        if(r != BIOIK_OK) return r;
        phases &= ~PH_MEMETIC;
    }
    if(ctx->serial_split && phases != PH_PREPARE)
    {
        int r = BIOIK_OK;
        for(int ph = 0; ph < 3 && r == BIOIK_OK; ph++)
        {
            if(!(phases & (1 << ph))) continue;
            Timed tp(ctx, st, 2 + ph);
            ctx->serial<<<sgrid, pl.block, pl.smem_bytes, st>>>(ctx->hP, S, step, 1 << ph);
            r = check_launch(ctx, "k_serial");
            tp.done();
        }
        return r;
    }
    Timed tm(ctx, st, 1);
    ctx->serial<<<sgrid, pl.block, pl.smem_bytes, st>>>(ctx->hP, S, step, phases);
    int r = check_launch(ctx, "k_serial");
    tm.done();
    return r;
}

// IKEvolution2::step for steps [s0, s1) of every run that is still going.  `last`: s1 is known to be the end of the solve (the
// approximator of a further step is not prepared).
int solve_steps(bioik_ctx* ctx, cudaStream_t st, int s0, int s1, bool last)
{
    RunPlan& R = ctx->run;
    if(!R.open) return fail(ctx, BIOIK_E_INVALID, "no solve in progress (bioik_begin)");
    if(s1 <= s0) return BIOIK_OK;
    int rc;
    if((rc = ensure_schedules(ctx, s1 + (ctx->S.islands > 1 ? (ctx->S.islands - 1) * ctx->S.island_stride : 0))) != BIOIK_OK) return rc;
    DState& S = ctx->S;
    S.gauss_off = ctx->d_gauss_off;
    S.rate_exp = ctx->d_rate_exp;
    const DProblem& P = ctx->hP;
    const int B = S.B, TPB = 128, warps_per_block = R.evolve_wpb;
    const int qblocks = (B + TPB - 1) / TPB, tblocks = (2 * B + TPB - 1) / TPB;
    if(!ctx->generic_now && R.persist)
    {
        // One launch per burst of steps.  With the driver's `finished` flag among islands that span several serial groups
        // (early_exit 2) the bursts end at the 4-step tests: a success recorded by one group must not be seen by a group that is
        // a step behind or ahead inside the same launch (the stepped path is in lock step by construction).
        const bool lockstep = S.early_exit == 2 && S.islands > PERSIST_GROUP_QUERIES;
        const int groups = (B + PERSIST_GROUP_QUERIES - 1) / PERSIST_GROUP_QUERIES;
        int a = s0;
        while(a < s1)
        {
            int b = std::min(s1, a + 64);
            if(lockstep) b = std::min(b, (a / 4 + 1) * 4);
            const bool last_here = last && b == s1;
            PersistArgs A;
            A.s0 = a, A.s1 = b, A.last = last_here ? 1 : 0, A.prepared = R.prepared ? 1 : 0, A.groups = groups, A.sm_count = ctx->sm_count;
            A.cap_e = (b - a) * B, A.cap_s = (b - a + 1) * groups;
            const size_t need = (size_t)A.cap_e + (size_t)A.cap_s;
            if(need > ctx->queue_slots || groups > ctx->gcount_cap || !ctx->d_qctr)
            {
                drop_graph(ctx);
                CU(ctx, cudaDeviceSynchronize());
                cudaFree(ctx->d_queue), cudaFree(ctx->d_gcount), cudaFree(ctx->d_qctr);
                ctx->d_queue = nullptr, ctx->d_gcount = nullptr, ctx->d_qctr = nullptr, ctx->queue_slots = 0, ctx->gcount_cap = 0;
                CU(ctx, cudaMalloc(&ctx->d_queue, need * 8));
                CU(ctx, cudaMalloc(&ctx->d_gcount, (size_t)groups * 4));
                CU(ctx, cudaMalloc(&ctx->d_qctr, PQ_INTS * 4));
                CU(ctx, cudaMemset(ctx->d_qctr, 0, PQ_INTS * 4));
                ctx->queue_slots = need, ctx->gcount_cap = groups;
            }
            A.slots_e = ctx->d_queue, A.slots_s = ctx->d_queue + A.cap_e, A.ctr = ctx->d_qctr, A.gcount = ctx->d_gcount;
            const int fill = std::max(std::max(A.cap_e, A.cap_s), groups);
            Timed tm(ctx, st, 0);
            k_persist_init<<<(fill + 255) / 256, 256, 0, st>>>(A, B);
            if((rc = check_launch(ctx, "k_persist_init")) != BIOIK_OK) return rc;
            int blocks = std::max(groups, (B + PERSIST_WARPS - 1) / PERSIST_WARPS);
            blocks = std::max(1, std::min(blocks, ctx->sm_count * R.persist_blocks_per_sm));
            R.persist<<<blocks, 32 * PERSIST_WARPS, R.persist_smem, st>>>(ctx->hP, ctx->dP, S, A, ctx->d_mtab);
            rc = check_launch(ctx, "k_persist");
            tm.done();
            if(rc != BIOIK_OK) return rc;
            R.prepared = !last_here;
            a = b;
        }
    }
    else if(!ctx->generic_now)
    {
        if(!R.prepared)
        {
            if((rc = launch_serial(ctx, st, s0, PH_PREPARE)) != BIOIK_OK) return rc;
            R.prepared = true;
        }
        for(int step = s0; step < s1; step++)
        {
            {
                const int tasks_per_block = warps_per_block * (R.fast ? 32 / R.evolve_lpt : 1);
                const int eb = (2 * B + tasks_per_block - 1) / tasks_per_block;
                Timed tm(ctx, st, 0);
                if(R.fast)
                    R.fast<<<eb, warps_per_block * 32, R.evolve_smem, st>>>(ctx->dP, S, step, ctx->d_mtab);
                else
                    k_evolve<<<eb, warps_per_block * 32, R.evolve_smem, st>>>(ctx->dP, S, step);
                rc = check_launch(ctx, "k_evolve");
                tm.done();
                if(rc != BIOIK_OK) return rc;
            }
            const bool prep = !(last && step + 1 == s1);
            const int phases = (S.memetic ? PH_MEMETIC : 0) | PH_SPECIES | (prep ? PH_PREPARE : 0);
            if((rc = launch_serial(ctx, st, step, phases)) != BIOIK_OK) return rc;
            R.prepared = prep;
        }
    }
    else
    {
        const int eblocks = (2 * B + warps_per_block - 1) / warps_per_block;
        for(int step = s0; step < s1; step++)
        {
            Timed t1(ctx, st, 1);
            k_prepare<<<tblocks, TPB, 0, st>>>(ctx->dP, S, step);
            if((rc = check_launch(ctx, "k_prepare")) != BIOIK_OK) return rc;
            t1.done();
            Timed t2(ctx, st, 0);
            k_evolve<<<eblocks, warps_per_block * 32, R.evolve_smem, st>>>(ctx->dP, S, step);
            if((rc = check_launch(ctx, "k_evolve")) != BIOIK_OK) return rc;
            t2.done();
            Timed t3(ctx, st, 1);
            if(S.memetic)
            {
                k_memetic<<<tblocks, TPB, 0, st>>>(ctx->dP, S, step);
                if((rc = check_launch(ctx, "k_memetic")) != BIOIK_OK) return rc;
            }
            k_species<<<qblocks, TPB, 0, st>>>(ctx->dP, S, step);
            if((rc = check_launch(ctx, "k_species")) != BIOIK_OK) return rc;
            t3.done();
        }
    }
    R.next_step = s1;
    return BIOIK_OK;
}

// number of runs that would execute step `step` (host polling between the driver's 4-step bursts); synchronises `st`
int count_active(bioik_ctx* ctx, cudaStream_t st, int step, int* out)
{
    if(!ctx->d_flag)
    {
        CU(ctx, cudaMalloc(&ctx->d_flag, 4));
        CU(ctx, cudaMallocHost(&ctx->h_flag, 4));
    }
    CU(ctx, cudaMemsetAsync(ctx->d_flag, 0, 4, st));
    k_count_active<<<(ctx->S.B + 255) / 256, 256, 0, st>>>(ctx->S, step, ctx->d_flag);
    int rc = check_launch(ctx, "k_count_active");
    if(rc != BIOIK_OK) return rc;
    CU(ctx, cudaMemcpyAsync(ctx->h_flag, ctx->d_flag, 4, cudaMemcpyDeviceToHost, st));
    CU(ctx, cudaStreamSynchronize(st));
    *out = *ctx->h_flag;
    return BIOIK_OK;
}

// after a stream synchronisation of a solve that used the persistent kernel: did its watchdog fire?
int check_watchdog(bioik_ctx* ctx)
{
    if(!ctx->run.persist || !ctx->d_qctr) return BIOIK_OK;
    int32_t fired = 0;
    CU(ctx, cudaMemcpy(&fired, ctx->d_qctr + PQ_ABORT, 4, cudaMemcpyDeviceToHost));
    if(fired) return fail(ctx, BIOIK_E_CUDA, "persistent solve kernel: watchdog fired (no work item became available for seconds); results are invalid");
    return BIOIK_OK;
}

// getSolution() of every run: full variable vector, primary fitness, success test, step count
int solve_finish(bioik_ctx* ctx, cudaStream_t st, double* d_osol, double* d_ofit, int32_t* d_osucc, int32_t* d_osteps)
{
    const int TPB = 128;
    k_finalize<<<(ctx->S.B + TPB - 1) / TPB, TPB, 0, st>>>(ctx->dP, ctx->S, d_osol, d_ofit, d_osucc, d_osteps);
    return check_launch(ctx, "k_finalize");
}

// enqueue a whole solve on `st`; all pointers are device pointers
int enqueue_solve(bioik_ctx* ctx, cudaStream_t st, int B, const double* d_gp, const double* d_seeds, const uint32_t* d_rs, int steps, int early_exit, double* d_osol, double* d_ofit, int32_t* d_osucc, int32_t* d_osteps)
{
    int rc = solve_begin(ctx, st, B, d_gp, d_seeds, d_rs, steps, early_exit, 0);
    if(rc != BIOIK_OK) return rc;
    if((rc = solve_steps(ctx, st, 0, steps, true)) != BIOIK_OK) return rc;
    return solve_finish(ctx, st, d_osol, d_ofit, d_osucc, d_osteps);
}

void drain_events_impl(bioik_ctx* ctx)
{
    for(auto& p : ctx->pending)
    {
        float ms = 0;
        cudaEventSynchronize(p.b);
        if(cudaEventElapsedTime(&ms, p.a, p.b) == cudaSuccess)
        {
            if(p.kind == 0)
                ctx->ms_evolve += ms, ctx->n_evolve++;
            else
            {
                ctx->ms_serial += ms, ctx->n_serial++;
                if(p.kind >= 2) ctx->ms_phase[p.kind - 2] += ms;
            }
        }
        ctx->pool.push_back(p);
    }
    ctx->pending.clear();
}
void drain_events(bioik_ctx* ctx) { drain_events_impl(ctx); }
} // namespace

extern "C" {

int bioik_abi_version(void) { return BIOIK_ABI_VERSION; }

const char* bioik_last_error(const bioik_ctx* ctx) { return ctx ? ctx->error.c_str() : g_create_error.c_str(); }

int bioik_create(const BioikRobot* robot, const BioikSolverCfg* cfg, bioik_ctx** out)
{
    Trace trace_("bioik_create");
    if(!robot || !cfg || !out) return fail(nullptr, BIOIK_E_INVALID, "null argument");
    *out = nullptr;
    if(cfg->population < 4 || cfg->population > 32 * EVOLVE_MAX_CPL) return fail(nullptr, BIOIK_E_LIMIT, "population must be in [4, 256]");
    if(cfg->generations < 1 || cfg->memetic_iters < 0) return fail(nullptr, BIOIK_E_INVALID, "bad generations / memetic_iters");
    if(cfg->memetic != 0 && cfg->memetic != 'q' && cfg->memetic != 'l') return fail(nullptr, BIOIK_E_INVALID, "memetic must be 0, 'q' or 'l'");
    if(robot->n_links < 1 || robot->n_vars < 1) return fail(nullptr, BIOIK_E_INVALID, "empty robot");
    bioik_ctx* ctx = new bioik_ctx();
    ctx->cfg = *cfg;
    {
        std::string err;
        int rc = intake_robot(robot, ctx->robot, err);
        if(rc != BIOIK_OK)
        {
            delete ctx;
            return fail(nullptr, rc, err);
        }
    }
    cudaError_t e = cudaSetDevice(cfg->device);
    if(e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
    if(e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->stream_cancel, cudaStreamNonBlocking);
    if(e == cudaSuccess) e = cudaMalloc(&ctx->d_cancel, 4);
    if(e == cudaSuccess) e = cudaMemset(ctx->d_cancel, 0, 4);
    if(e == cudaSuccess) e = cudaMallocHost(&ctx->h_one, 4);
    if(e == cudaSuccess) *ctx->h_one = 1;
    if(e == cudaSuccess) e = cudaMalloc(&ctx->d_uniform, sizeof(double) * 1024 * 1024 * 8);
    if(e == cudaSuccess) e = cudaMalloc(&ctx->d_gauss, sizeof(double) * 1024 * 1024 * 8);
    if(e == cudaSuccess) e = cudaMalloc(&ctx->dP, sizeof(DProblem));
    if(e == cudaSuccess)
    {
        std::vector<double> u, g;
        make_tables(cfg->table_seed, u, g);
        for(double v : g) ctx->gauss_absmax = std::max(ctx->gauss_absmax, std::fabs(v));
        e = cudaMemcpy(ctx->d_uniform, u.data(), u.size() * 8, cudaMemcpyHostToDevice);
        if(e == cudaSuccess) e = cudaMemcpy(ctx->d_gauss, g.data(), g.size() * 8, cudaMemcpyHostToDevice);
    }
    if(e != cudaSuccess)
    {
        std::string msg = std::string("CUDA initialisation failed (no CPU fallback exists): ") + cudaGetErrorString(e);
        bioik_destroy(ctx);
        return fail(nullptr, BIOIK_E_CUDA, msg);
    }
    memset(&ctx->S, 0, sizeof(ctx->S));
    cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, cfg->device);
    {
        const char* fg = getenv("BIOIK_FORCE_GENERIC");
        ctx->force_generic = fg && fg[0] == '1';
        const char* ng = getenv("BIOIK_NO_GRAPH");
        ctx->use_graphs = !(ng && ng[0] == '1');
        const char* spf = getenv("BIOIK_SERIAL_PLAN");
        if(spf) ctx->serial_plan_force = atoi(spf);
        const char* lp = getenv("BIOIK_EVOLVE_LPT");
        if(lp && atoi(lp) > 0) ctx->lpt_want = atoi(lp);
        const char* ch = getenv("BIOIK_EVOLVE_CH");
        if(ch && atoi(ch) > 0) ctx->ch_cap = atoi(ch);
        const char* mg = getenv("BIOIK_MEMETIC_GROUP");
        ctx->memetic_group = mg ? (mg[0] == '0' ? 0 : 1) : -1;
        const char* pm = getenv("BIOIK_PERSIST");
        if(pm) ctx->persist_mode = atoi(pm);
        const char* sp = getenv("BIOIK_SERIAL_SPLIT");
        ctx->serial_split = sp && sp[0] == '1';
    }
    *out = ctx;
    return BIOIK_OK;
}

void bioik_destroy(bioik_ctx* ctx)
{
    Trace trace_("bioik_destroy");
    if(!ctx) return;
    cudaSetDevice(ctx->cfg.device);
    cudaDeviceSynchronize();
    if(ctx->graph_exec) cudaGraphExecDestroy(ctx->graph_exec);
    for(auto& p : ctx->pending) cudaEventDestroy(p.a), cudaEventDestroy(p.b);
    for(auto& p : ctx->pool) cudaEventDestroy(p.a), cudaEventDestroy(p.b);
    cudaFree(ctx->d_uniform), cudaFree(ctx->d_gauss), cudaFree(ctx->dP), cudaFree(ctx->d_gauss_off), cudaFree(ctx->d_rate_exp), cudaFree(ctx->d_mtab), cudaFree(ctx->state_block);
    cudaFree(ctx->d_gp), cudaFree(ctx->d_seeds), cudaFree(ctx->d_rs), cudaFree(ctx->d_osol), cudaFree(ctx->d_ofit), cudaFree(ctx->d_osucc), cudaFree(ctx->d_osteps), cudaFree(ctx->d_default_gp);
    cudaFree(ctx->d_flag), cudaFree(ctx->d_cancel);
    cudaFree(ctx->d_queue), cudaFree(ctx->d_qctr), cudaFree(ctx->d_gcount);
    if(ctx->h_one) cudaFreeHost(ctx->h_one);
    if(ctx->stream_cancel) cudaStreamDestroy(ctx->stream_cancel);
    if(ctx->h_flag) cudaFreeHost(ctx->h_flag);
    cudaFree(ctx->d_q_gp), cudaFree(ctx->d_q_seeds), cudaFree(ctx->d_q_sol), cudaFree(ctx->d_q_fit), cudaFree(ctx->d_q_succ), cudaFree(ctx->d_q_island), cudaFree(ctx->d_q_steps);
    if(ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

int bioik_set_problem(bioik_ctx* ctx, const BioikProblem* problem)
{
    Trace trace_("bioik_set_problem");
    if(!ctx || !problem) return fail(ctx, BIOIK_E_INVALID, "null argument");
    CU(ctx, cudaSetDevice(ctx->cfg.device));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->has_problem = false;
    int rc = build_problem(ctx->robot, problem, ctx->hP, ctx->error);
    if(rc != BIOIK_OK) return rc;
    CU(ctx, cudaMemcpy(ctx->dP, &ctx->hP, sizeof(DProblem), cudaMemcpyHostToDevice));

    std::vector<double> gp((size_t)problem->n_goals * GOAL_NPARAM);
    for(int g = 0; g < problem->n_goals; g++)
        for(int k = 0; k < GOAL_NPARAM; k++) gp[(size_t)g * GOAL_NPARAM + k] = problem->goals[g].p[k];
    cudaFree(ctx->d_default_gp);
    ctx->d_default_gp = nullptr;
    CU(ctx, cudaMalloc(&ctx->d_default_gp, gp.size() * 8));
    CU(ctx, cudaMemcpy(ctx->d_default_gp, gp.data(), gp.size() * 8, cudaMemcpyHostToDevice));
    // state/staging/schedules depend on the problem shape: drop them
    cudaFree(ctx->state_block);
    ctx->state_block = nullptr;
    ctx->capB = 0;
    cudaFree(ctx->d_gp), cudaFree(ctx->d_seeds), cudaFree(ctx->d_rs), cudaFree(ctx->d_osol), cudaFree(ctx->d_ofit), cudaFree(ctx->d_osucc), cudaFree(ctx->d_osteps);
    ctx->d_gp = ctx->d_seeds = ctx->d_osol = ctx->d_ofit = nullptr;
    ctx->d_rs = nullptr;
    ctx->d_osucc = ctx->d_osteps = nullptr;
    ctx->stageB = 0;
    ctx->queryQ = 0;
    ctx->sched_steps = -1;
    drop_graph(ctx);
    ctx->run = RunPlan();
    ctx->has_problem = true;
    return BIOIK_OK;
}

int bioik_solve_batch_device(bioik_ctx* ctx, int32_t B, const double* d_goal_params, const double* d_seeds, const uint32_t* d_rng_seeds, int32_t steps, int32_t early_exit, double* d_out_solutions, double* d_out_fitness,
                             int32_t* d_out_success, int32_t* d_out_steps, void* cuda_stream)
{
    Trace trace_("bioik_solve_batch_device");
    if(!ctx) return BIOIK_E_INVALID;
    CU(ctx, cudaSetDevice(ctx->cfg.device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
    CU(ctx, cudaMemsetAsync(ctx->d_cancel, 0, 4, st)); // IKParallel::solve: canceled = false at the start of every solve (src/ik_parallel.h:211-212)
    return enqueue_solve(ctx, st, B, d_goal_params, d_seeds, d_rng_seeds, steps, early_exit, d_out_solutions, d_out_fitness, d_out_success, d_out_steps);
}

int bioik_solve_batch(bioik_ctx* ctx, int32_t B, const double* goal_params, const double* seeds, const uint32_t* rng_seeds, int32_t steps, int32_t early_exit, double* out_solutions, double* out_fitness, int32_t* out_success,
                      int32_t* out_steps)
{
    Trace trace_("bioik_solve_batch");
    if(!ctx) return BIOIK_E_INVALID;
    if(!ctx->has_problem) return fail(ctx, BIOIK_E_NO_PROBLEM, "bioik_set_problem has not been called");
    if(B <= 0 || !seeds || !rng_seeds) return fail(ctx, BIOIK_E_INVALID, "bad solve arguments");
    CU(ctx, cudaSetDevice(ctx->cfg.device));
    CU(ctx, cudaMemsetAsync(ctx->d_cancel, 0, 4, ctx->stream)); // IKParallel::solve: canceled = false (src/ik_parallel.h:211-212)
    int rc = ensure_staging(ctx, B);
    if(rc != BIOIK_OK) return rc;
    const DProblem& P = ctx->hP;
    cudaStream_t st = ctx->stream;
    if(goal_params) CU(ctx, cudaMemcpyAsync(ctx->d_gp, goal_params, (size_t)B * P.G * GOAL_NPARAM * 8, cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemcpyAsync(ctx->d_seeds, seeds, (size_t)B * P.n_vars * 8, cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemcpyAsync(ctx->d_rs, rng_seeds, (size_t)B * 4, cudaMemcpyHostToDevice, st));
    // Repeated solves of one shape replay a CUDA graph of the ~50 kernel launches (first call eager: it sizes the
    // state; second call captures; later calls replay).  Per-launch timing and graphs exclude each other.
    const int has_gp = goal_params ? 1 : 0;
    const bool same_shape = ctx->graph_B == B && ctx->graph_steps == steps && ctx->graph_early == early_exit && ctx->graph_gp == has_gp;
    if(ctx->use_graphs && !ctx->timing && same_shape && ctx->graph_exec)
    {
        CU(ctx, cudaGraphLaunch(ctx->graph_exec, st));
        ctx->launches += ctx->graph_launches;
    }
    else if(ctx->use_graphs && !ctx->timing && same_shape)
    {
        cudaGraph_t graph = nullptr;
        CU(ctx, cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        ctx->capturing = true;
        const int64_t l0 = ctx->launches;
        rc = enqueue_solve(ctx, st, B, goal_params ? ctx->d_gp : nullptr, ctx->d_seeds, ctx->d_rs, steps, early_exit, ctx->d_osol, ctx->d_ofit, ctx->d_osucc, ctx->d_osteps);
        ctx->capturing = false;
        cudaError_t ce = cudaStreamEndCapture(st, &graph);
        if(rc != BIOIK_OK)
        {
            if(graph) cudaGraphDestroy(graph);
            return rc;
        }
        if(ce != cudaSuccess) return fail(ctx, BIOIK_E_CUDA, std::string("cudaStreamEndCapture: ") + cudaGetErrorString(ce));
        ctx->graph_launches = ctx->launches - l0;
        ce = cudaGraphInstantiate(&ctx->graph_exec, graph, 0);
        cudaGraphDestroy(graph);
        if(ce != cudaSuccess)
        {
            ctx->graph_exec = nullptr;
            return fail(ctx, BIOIK_E_CUDA, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(ce));
        }
        CU(ctx, cudaGraphLaunch(ctx->graph_exec, st));
    }
    else
    {
        drop_graph(ctx);
        rc = enqueue_solve(ctx, st, B, goal_params ? ctx->d_gp : nullptr, ctx->d_seeds, ctx->d_rs, steps, early_exit, ctx->d_osol, ctx->d_ofit, ctx->d_osucc, ctx->d_osteps);
        if(rc != BIOIK_OK) return rc;
        ctx->graph_B = B, ctx->graph_steps = steps, ctx->graph_early = early_exit, ctx->graph_gp = has_gp;
    }
    if(out_solutions) CU(ctx, cudaMemcpyAsync(out_solutions, ctx->d_osol, (size_t)B * P.n_vars * 8, cudaMemcpyDeviceToHost, st));
    if(out_fitness) CU(ctx, cudaMemcpyAsync(out_fitness, ctx->d_ofit, (size_t)B * 8, cudaMemcpyDeviceToHost, st));
    if(out_success) CU(ctx, cudaMemcpyAsync(out_success, ctx->d_osucc, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
    if(out_steps) CU(ctx, cudaMemcpyAsync(out_steps, ctx->d_osteps, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
    CU(ctx, cudaStreamSynchronize(st));
    return check_watchdog(ctx);
}

int bioik_cancel(bioik_ctx* ctx)
{
    if(!ctx || !ctx->d_cancel) return BIOIK_E_INVALID;
    // may be called from another thread while a solve is running: touches nothing of the context but this stream
    if(cudaSetDevice(ctx->cfg.device) != cudaSuccess) return BIOIK_E_CUDA;
    if(cudaMemcpyAsync(ctx->d_cancel, ctx->h_one, 4, cudaMemcpyHostToDevice, ctx->stream_cancel) != cudaSuccess) return BIOIK_E_CUDA;
    return BIOIK_OK;
}

int bioik_set_option(bioik_ctx* ctx, int32_t option, int32_t value)
{
    if(!ctx) return BIOIK_E_INVALID;
    switch(option)
    {
    case BIOIK_OPT_REFERENCE_STALE_TIPS:
        ctx->stale_tips = value != 0;
        drop_graph(ctx);
        return BIOIK_OK;
    case BIOIK_OPT_ISLAND_STREAM_STRIDE:
        if(value < 0 || value > 64) return fail(ctx, BIOIK_E_INVALID, "BIOIK_OPT_ISLAND_STREAM_STRIDE must be in [0, 64]");
        ctx->island_stride = value;
        drop_graph(ctx);
        return BIOIK_OK;
    default: return fail(ctx, BIOIK_E_INVALID, "unknown option");
    }
}

int bioik_begin(bioik_ctx* ctx, int32_t Q, int32_t islands, const double* goal_params, const double* seeds, const uint32_t* rng_seeds, int32_t max_steps, int32_t early_exit)
{
    Trace trace_("bioik_begin");
    if(!ctx) return BIOIK_E_INVALID;
    if(!ctx->has_problem) return fail(ctx, BIOIK_E_NO_PROBLEM, "bioik_set_problem has not been called");
    if(Q <= 0 || islands <= 0 || max_steps < 0 || !seeds || !rng_seeds || (int64_t)Q * islands > (int64_t)INT32_MAX / 4) return fail(ctx, BIOIK_E_INVALID, "bad bioik_begin arguments");
    CU(ctx, cudaSetDevice(ctx->cfg.device));
    ctx->run.open = false;
    CU(ctx, cudaMemsetAsync(ctx->d_cancel, 0, 4, ctx->stream)); // IKParallel::solve: canceled = false (src/ik_parallel.h:211-212)
    const int B = Q * islands;
    int rc = ensure_staging(ctx, B);
    if(rc != BIOIK_OK) return rc;
    const DProblem& P = ctx->hP;
    cudaStream_t st = ctx->stream;
    if(Q > ctx->queryQ)
    {
        CU(ctx, cudaStreamSynchronize(st));
        cudaFree(ctx->d_q_gp), cudaFree(ctx->d_q_seeds), cudaFree(ctx->d_q_sol), cudaFree(ctx->d_q_fit), cudaFree(ctx->d_q_succ), cudaFree(ctx->d_q_island), cudaFree(ctx->d_q_steps);
        ctx->d_q_gp = ctx->d_q_seeds = ctx->d_q_sol = ctx->d_q_fit = nullptr, ctx->d_q_succ = ctx->d_q_island = ctx->d_q_steps = nullptr;
        ctx->queryQ = 0;
        CU(ctx, cudaMalloc(&ctx->d_q_gp, (size_t)Q * P.G * GOAL_NPARAM * 8 + 8));
        CU(ctx, cudaMalloc(&ctx->d_q_seeds, (size_t)Q * P.n_vars * 8));
        CU(ctx, cudaMalloc(&ctx->d_q_sol, (size_t)Q * P.n_vars * 8));
        CU(ctx, cudaMalloc(&ctx->d_q_fit, (size_t)Q * 8));
        CU(ctx, cudaMalloc(&ctx->d_q_succ, (size_t)Q * 4));
        CU(ctx, cudaMalloc(&ctx->d_q_island, (size_t)Q * 4));
        CU(ctx, cudaMalloc(&ctx->d_q_steps, (size_t)Q * 4));
        ctx->queryQ = Q;
    }
    const int per_gp = P.G * GOAL_NPARAM, per_seed = P.n_vars;
    if(goal_params) CU(ctx, cudaMemcpyAsync(ctx->d_q_gp, goal_params, (size_t)Q * per_gp * 8, cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemcpyAsync(ctx->d_q_seeds, seeds, (size_t)Q * per_seed * 8, cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemcpyAsync(ctx->d_rs, rng_seeds, (size_t)B * 4, cudaMemcpyHostToDevice, st));
    {
        const size_t total = (size_t)B * std::max(per_gp, per_seed);
        k_expand_islands<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(Q, islands, per_gp, per_seed, goal_params ? ctx->d_q_gp : nullptr, ctx->d_q_seeds, ctx->d_gp, ctx->d_seeds);
        if((rc = check_launch(ctx, "k_expand_islands")) != BIOIK_OK) return rc;
    }
    drop_graph(ctx); // the staging buffers are shared with the cached solve_batch graph
    // no step budget: the driver's test still runs after every 4th step, there is just no "last step" (src/ik_parallel.h:165-181)
    rc = solve_begin(ctx, st, B, goal_params ? ctx->d_gp : nullptr, ctx->d_seeds, ctx->d_rs, max_steps > 0 ? max_steps : INT32_MAX, early_exit, islands);
    if(rc != BIOIK_OK) return rc;
    ctx->run.Q = Q, ctx->run.islands = islands;
    CU(ctx, cudaStreamSynchronize(st)); // the caller's host buffers are free again
    return BIOIK_OK;
}

int bioik_step(bioik_ctx* ctx, int32_t nsteps, int32_t* out_active)
{
    Trace trace_("bioik_step");
    if(!ctx) return BIOIK_E_INVALID;
    if(!ctx->run.open || ctx->run.islands <= 0) return fail(ctx, BIOIK_E_INVALID, "bioik_step without bioik_begin");
    if(nsteps < 0) return fail(ctx, BIOIK_E_INVALID, "negative step count");
    CU(ctx, cudaSetDevice(ctx->cfg.device));
    const int s0 = ctx->run.next_step, total = ctx->S.total_steps;
    const int s1 = (int)std::min<int64_t>((int64_t)s0 + nsteps, total);
    int rc = solve_steps(ctx, ctx->stream, s0, s1, s1 == total);
    if(rc != BIOIK_OK) return rc;
    if(out_active)
    {
        int active = 0;
        if(s1 < total && (rc = count_active(ctx, ctx->stream, s1, &active)) != BIOIK_OK) return rc;
        *out_active = active;
    }
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    return check_watchdog(ctx);
}

int bioik_get_solution(bioik_ctx* ctx, int32_t wrap, double* out_solutions, double* out_fitness, int32_t* out_success, int32_t* out_island, int32_t* out_steps)
{
    Trace trace_("bioik_get_solution");
    if(!ctx) return BIOIK_E_INVALID;
    if(!ctx->run.open || ctx->run.islands <= 0) return fail(ctx, BIOIK_E_INVALID, "bioik_get_solution without bioik_begin");
    if(!out_solutions) return fail(ctx, BIOIK_E_INVALID, "out_solutions is required");
    CU(ctx, cudaSetDevice(ctx->cfg.device));
    const DProblem& P = ctx->hP;
    cudaStream_t st = ctx->stream;
    const int Q = ctx->run.Q, islands = ctx->run.islands;
    int rc = solve_finish(ctx, st, ctx->d_osol, ctx->d_ofit, ctx->d_osucc, ctx->d_osteps);
    if(rc != BIOIK_OK) return rc;
    // (without per-query parameters solve_begin has broadcast the defaults into d_gp)
    k_select_islands<<<(Q + 127) / 128, 128, 0, st>>>(ctx->dP, Q, islands, ctx->d_gp, ctx->d_seeds, ctx->d_osol, ctx->d_ofit, ctx->d_osucc, ctx->d_osteps, wrap, ctx->d_q_sol, ctx->d_q_fit, ctx->d_q_succ, ctx->d_q_island,
                                                      ctx->d_q_steps);
    if((rc = check_launch(ctx, "k_select_islands")) != BIOIK_OK) return rc;
    CU(ctx, cudaMemcpyAsync(out_solutions, ctx->d_q_sol, (size_t)Q * P.n_vars * 8, cudaMemcpyDeviceToHost, st));
    if(out_fitness) CU(ctx, cudaMemcpyAsync(out_fitness, ctx->d_q_fit, (size_t)Q * 8, cudaMemcpyDeviceToHost, st));
    if(out_success) CU(ctx, cudaMemcpyAsync(out_success, ctx->d_q_succ, (size_t)Q * 4, cudaMemcpyDeviceToHost, st));
    if(out_island) CU(ctx, cudaMemcpyAsync(out_island, ctx->d_q_island, (size_t)Q * 4, cudaMemcpyDeviceToHost, st));
    if(out_steps) CU(ctx, cudaMemcpyAsync(out_steps, ctx->d_q_steps, (size_t)Q * 4, cudaMemcpyDeviceToHost, st));
    CU(ctx, cudaStreamSynchronize(st));
    return BIOIK_OK;
}

int bioik_solve_islands(bioik_ctx* ctx, int32_t Q, int32_t islands, const double* goal_params, const double* seeds, const uint32_t* rng_seeds, int32_t steps, int32_t early_exit, int32_t wrap, double* out_solutions,
                        double* out_fitness, int32_t* out_success, int32_t* out_island, int32_t* out_steps)
{
    Trace trace_("bioik_solve_islands");
    if(!ctx) return BIOIK_E_INVALID;
    if(!out_solutions || steps < 0) return fail(ctx, BIOIK_E_INVALID, "bad solve_islands arguments");
    int rc = bioik_begin(ctx, Q, islands, goal_params, seeds, rng_seeds, steps, early_exit);
    if(rc != BIOIK_OK) return rc;
    if(steps == 0) ctx->S.total_steps = 0; // bioik_begin reads 0 as "no budget"
    // the driver's 4-step bursts (src/ik_parallel.h:165-168); with an early exit the host asks after each of them whether any run
    // is still going and stops enqueueing when none is (every kernel would return at once, but the launches add up)
    for(int s = 0; s < steps; s += 4)
    {
        int32_t active = 1;
        if((rc = bioik_step(ctx, std::min(4, steps - s), early_exit ? &active : nullptr)) != BIOIK_OK) return rc;
        if(early_exit && !active) break;
    }
    return bioik_get_solution(ctx, wrap, out_solutions, out_fitness, out_success, out_island, out_steps);
}

int bioik_solve_batch_trace(bioik_ctx* ctx, int32_t B, const double* goal_params, const double* seeds, const uint32_t* rng_seeds, int32_t steps, double* out_genes, double* out_gradients, double* out_species_fitness,
                            double* out_solutions, double* out_fitness)
{
    int rc = bioik_solve_batch(ctx, B, goal_params, seeds, rng_seeds, steps, 0, out_solutions, out_fitness, nullptr, nullptr);
    if(rc != BIOIK_OK) return rc;
    size_t n = ctx->hP.n;
    if(out_genes) CU(ctx, cudaMemcpy(out_genes, ctx->S.genes, (size_t)B * 4 * n * 8, cudaMemcpyDeviceToHost));
    if(out_gradients) CU(ctx, cudaMemcpy(out_gradients, ctx->S.grads, (size_t)B * 4 * n * 8, cudaMemcpyDeviceToHost));
    if(out_species_fitness) CU(ctx, cudaMemcpy(out_species_fitness, ctx->S.sfit, (size_t)B * 2 * 8, cudaMemcpyDeviceToHost));
    return BIOIK_OK;
}

int bioik_synchronize(bioik_ctx* ctx)
{
    if(!ctx) return BIOIK_E_INVALID;
    CU(ctx, cudaSetDevice(ctx->cfg.device));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    return BIOIK_OK;
}

int bioik_fk_batch(bioik_ctx* ctx, int32_t B, const double* variables, double* out_tip_frames)
{
    if(!ctx) return BIOIK_E_INVALID;
    if(!ctx->has_problem) return fail(ctx, BIOIK_E_NO_PROBLEM, "bioik_set_problem has not been called");
    CU(ctx, cudaSetDevice(ctx->cfg.device));
    const DProblem& P = ctx->hP;
    double *dv = nullptr, *dt = nullptr;
    CU(ctx, cudaMalloc(&dv, (size_t)B * P.n_vars * 8));
    CU(ctx, cudaMalloc(&dt, (size_t)B * P.T * 7 * 8));
    CU(ctx, cudaMemcpyAsync(dv, variables, (size_t)B * P.n_vars * 8, cudaMemcpyHostToDevice, ctx->stream));
    k_fk_batch<<<(B + 127) / 128, 128, 0, ctx->stream>>>(ctx->dP, B, dv, dt);
    int rc = check_launch(ctx, "k_fk_batch");
    if(rc == BIOIK_OK)
    {
        cudaError_t e = cudaMemcpyAsync(out_tip_frames, dt, (size_t)B * P.T * 7 * 8, cudaMemcpyDeviceToHost, ctx->stream);
        if(e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if(e != cudaSuccess) rc = fail(ctx, BIOIK_E_CUDA, cudaGetErrorString(e));
    }
    cudaFree(dv), cudaFree(dt);
    return rc;
}

int bioik_approx_batch(bioik_ctx* ctx, int32_t B, const double* variables, double* out_delta_frames)
{
    if(!ctx) return BIOIK_E_INVALID;
    if(!ctx->has_problem) return fail(ctx, BIOIK_E_NO_PROBLEM, "bioik_set_problem has not been called");
    CU(ctx, cudaSetDevice(ctx->cfg.device));
    const DProblem& P = ctx->hP;
    double *dv = nullptr, *dd = nullptr;
    size_t dn = (size_t)B * P.T * P.n * 7 * 8;
    CU(ctx, cudaMalloc(&dv, (size_t)B * P.n_vars * 8));
    CU(ctx, cudaMalloc(&dd, dn));
    CU(ctx, cudaMemcpyAsync(dv, variables, (size_t)B * P.n_vars * 8, cudaMemcpyHostToDevice, ctx->stream));
    k_approx_batch<<<(B + 127) / 128, 128, 0, ctx->stream>>>(ctx->dP, B, dv, dd);
    int rc = check_launch(ctx, "k_approx_batch");
    if(rc == BIOIK_OK)
    {
        cudaError_t e = cudaMemcpyAsync(out_delta_frames, dd, dn, cudaMemcpyDeviceToHost, ctx->stream);
        if(e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if(e != cudaSuccess) rc = fail(ctx, BIOIK_E_CUDA, cudaGetErrorString(e));
    }
    cudaFree(dv), cudaFree(dd);
    return rc;
}

int bioik_approx_fitness_batch(bioik_ctx* ctx, int32_t B, int32_t M, const double* goal_params, const double* seeds, const double* base_variables, const double* genotypes, double* out_primary, double* out_secondary)
{
    if(!ctx) return BIOIK_E_INVALID;
    if(!ctx->has_problem) return fail(ctx, BIOIK_E_NO_PROBLEM, "bioik_set_problem has not been called");
    CU(ctx, cudaSetDevice(ctx->cfg.device));
    const DProblem& P = ctx->hP;
    size_t ngp = (size_t)B * P.G * GOAL_NPARAM, nv = (size_t)B * P.n_vars, ng = (size_t)B * M * P.n, nf = (size_t)B * M;
    std::vector<double> gp_host;
    if(!goal_params)
    {
        gp_host.resize(ngp);
        std::vector<double> def((size_t)P.G * GOAL_NPARAM);
        cudaMemcpy(def.data(), ctx->d_default_gp, def.size() * 8, cudaMemcpyDeviceToHost);
        for(int b = 0; b < B; b++) std::copy(def.begin(), def.end(), gp_host.begin() + (size_t)b * def.size());
        goal_params = gp_host.data();
    }
    double *d_gp = nullptr, *d_seed = nullptr, *d_base = nullptr, *d_gen = nullptr, *d_p = nullptr, *d_s = nullptr, *d_scr = nullptr;
    CU(ctx, cudaMalloc(&d_gp, ngp * 8));
    CU(ctx, cudaMalloc(&d_seed, nv * 8));
    CU(ctx, cudaMalloc(&d_base, nv * 8));
    CU(ctx, cudaMalloc(&d_gen, ng * 8));
    CU(ctx, cudaMalloc(&d_p, nf * 8));
    CU(ctx, cudaMalloc(&d_s, nf * 8));
    CU(ctx, cudaMalloc(&d_scr, nf * P.T * P.n * 7 * 8));
    cudaStream_t st = ctx->stream;
    CU(ctx, cudaMemcpyAsync(d_gp, goal_params, ngp * 8, cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemcpyAsync(d_seed, seeds, nv * 8, cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemcpyAsync(d_base, base_variables, nv * 8, cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemcpyAsync(d_gen, genotypes, ng * 8, cudaMemcpyHostToDevice, st));
    k_approx_fitness<<<(int)((nf + 127) / 128), 128, 0, st>>>(ctx->dP, B, M, d_gp, d_seed, d_base, d_gen, d_p, d_s, d_scr);
    int rc = check_launch(ctx, "k_approx_fitness");
    if(rc == BIOIK_OK)
    {
        cudaError_t e = cudaSuccess;
        if(out_primary) e = cudaMemcpyAsync(out_primary, d_p, nf * 8, cudaMemcpyDeviceToHost, st);
        if(e == cudaSuccess && out_secondary) e = cudaMemcpyAsync(out_secondary, d_s, nf * 8, cudaMemcpyDeviceToHost, st);
        if(e == cudaSuccess) e = cudaStreamSynchronize(st);
        if(e != cudaSuccess) rc = fail(ctx, BIOIK_E_CUDA, cudaGetErrorString(e));
    }
    cudaFree(d_gp), cudaFree(d_seed), cudaFree(d_base), cudaFree(d_gen), cudaFree(d_p), cudaFree(d_s), cudaFree(d_scr);
    return rc;
}

int bioik_pack_results_device(bioik_ctx* ctx, int32_t B, const double* d_solutions, const double* d_fitness, const int32_t* d_success, const int32_t* d_steps, double* d_slab, void* cuda_stream)
{
    if(!ctx) return BIOIK_E_INVALID;
    if(!ctx->has_problem) return fail(ctx, BIOIK_E_NO_PROBLEM, "bioik_set_problem has not been called");
    if(B <= 0 || !d_solutions || !d_fitness || !d_success || !d_steps || !d_slab) return fail(ctx, BIOIK_E_INVALID, "bad pack arguments");
    CU(ctx, cudaSetDevice(ctx->cfg.device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
    const size_t total = (size_t)B * (ctx->hP.n_vars + 3);
    k_pack_results<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(B, ctx->hP.n_vars, d_solutions, d_fitness, d_success, d_steps, d_slab);
    return check_launch(ctx, "k_pack_results");
}

const char* bioik_kernel_name(const bioik_ctx* ctx) { return ctx ? ctx->run.dominant : ""; }

int64_t bioik_launch_count(const bioik_ctx* ctx) { return ctx ? ctx->launches : 0; }

int bioik_kernel_time(bioik_ctx* ctx, int32_t reset, double* out_ms_evolve, int64_t* out_launches_evolve, double* out_ms_serial, int64_t* out_launches_serial)
{
    if(!ctx) return BIOIK_E_INVALID;
    CU(ctx, cudaSetDevice(ctx->cfg.device));
    CU(ctx, cudaDeviceSynchronize());
    drain_events(ctx);
#ifdef BIOIK_PERSIST_STATS
    if(ctx->d_qctr)
    {
        unsigned long long st[8];
        cudaMemcpy(st, ctx->d_qctr + PQ_STATS, sizeof(st), cudaMemcpyDeviceToHost);
        if(st[7])
            fprintf(stderr, "[bioik] persistent kernel, per warp-launch averages over %llu warp-launches: resident %.0f cycles = evolve %.0f (%.2f items of %.0f) + serial %.0f (%.2f items of %.0f) + idle %.0f (%.1f polls)\n", st[7],
                    (double)st[6] / st[7], (double)st[0] / st[7], (double)st[3] / st[7], st[3] ? (double)st[0] / st[3] : 0.0, (double)st[1] / st[7], (double)st[4] / st[7], st[4] ? (double)st[1] / st[4] : 0.0,
                    (double)st[2] / st[7], (double)st[5] / st[7]);
        if(reset) cudaMemset(ctx->d_qctr + PQ_STATS, 0, sizeof(st));
    }
#endif
    if(ctx->serial_split && ctx->n_serial)
        fprintf(stderr, "[bioik] serial phases (ms total): memetic %.3f species %.3f prepare %.3f over %lld launches\n", ctx->ms_phase[0], ctx->ms_phase[1], ctx->ms_phase[2], (long long)ctx->n_serial);
    if(reset) ctx->ms_phase[0] = ctx->ms_phase[1] = ctx->ms_phase[2] = 0;
    ctx->timing = (reset != 2); // the first call switches per-launch timing on; reset == 2 switches it off again
    if(out_ms_evolve) *out_ms_evolve = ctx->ms_evolve;
    if(out_launches_evolve) *out_launches_evolve = ctx->n_evolve;
    if(out_ms_serial) *out_ms_serial = ctx->ms_serial;
    if(out_launches_serial) *out_launches_serial = ctx->n_serial;
    if(reset)
    {
        ctx->ms_evolve = ctx->ms_serial = 0;
        ctx->n_evolve = ctx->n_serial = 0;
    }
    return BIOIK_OK;
}
}
