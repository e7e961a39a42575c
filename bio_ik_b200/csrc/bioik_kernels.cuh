// bioik_kernels.cuh — sm_90a kernels of the batched bio2 / bio2_memetic solver.
//
// Work decomposition (DESIGN.md §4): a QUERY is one independent IK problem; a TASK is
// (query, species slot).  The two species of a query never interact inside a step()
// (src/ik_evolution_2.cpp:332-602), only in the species block (:604-645), so they run as
// independent tasks.  Per step:
//   k_prepare  thread/task   exact FK + Jacobian + delta frames at individuals[0]   (:341-346)
//   k_evolve   warp/task     `generations` x {reproduce, phenotype, fitness, select} (:351-432)
//   k_memetic  thread/task   quadratic / linear line search on individuals[0]      (:436-570)
//   k_species  thread/query  exact fitness, species sort, wipeout, solution update (:604-645)
//                            + the driver's success test (src/ik_parallel.h:173-181)
#pragma once

#include "bioik_dev.cuh"

namespace bioik
{

// Per-batch solver state in HBM.  Layout: one contiguous record per query for every
// field ("array of per-query records"), fields in separate arrays.
struct DState
{
    int32_t B, C, gens, memetic, memetic_iters, total_steps, early_exit, islands; // islands > 1: run q is island q % islands of query q / islands
    int32_t island_stride; // islands > 1: island k reads the query-independent random streams `k * island_stride` steps ahead (0: all islands share them)
    // inputs
    const double* goal_params; // [B][G][NPARAM]
    const double* seeds;       // [B][n_vars]
    const uint32_t* rng_seeds; // [B]
    // solver state
    double* genes;     // [B][2 slots][2 individuals][n]
    double* grads;     // [B][2][2][n]
    double* sfit;      // [B][2] Species::fitness
    int32_t* impr;     // [B][2] Species::improved
    double* sol;       // [B][n] solution (active part)
    double* solfit;    // [B]
    uint32_t* rng;     // [B] minstd state
    int32_t* done;     // [B]
    int32_t* steps;    // [B] step() calls executed
    int32_t* success;  // [B]
    int32_t* ccount;   // [B][2][gens] pre-selection child_count (only with secondary goals)
    double* carry;     // [B][T][7] reference-quirk mode: frames left in the solver's phenotypes3 (identity at the start)
    const volatile int32_t* cancel; // device flag set by bioik_cancel (the reference's `volatile int canceled`, src/ik_base.h:143): every run counts as done
    int32_t* qstep;    // [B / islands] step count at which the first island of the query passed the success test (INT32_MAX: none yet)
    // approximator of the current step
    double* base;  // [B][2][n]
    double* tip0;  // [B][2][T][7]
    double* delta; // [B][2][T][n][7]
    // shared lookup tables / schedules
    const double* uniform;     // [2^23]
    const double* gauss;       // [2^23]
    double gauss_absmax;       // max |gauss[i]| over the table: bounds every mutation term (clamp elision in the generation kernel)
    const int32_t* gauss_off;  // [total_steps*2*gens] slab start of each reproduce() call
    const uint8_t* rate_exp;   // [total_steps*2*gens][C-2] fast_random_index(16) per child
};

// A run is over when its own early exit fired, or - early_exit == 2, the islands of one query - when a sibling island passed
// the driver's success test at an EARLIER check: IKParallel's `finished` flag (src/ik_parallel.h:160,164,171,180), which
// makes every other solver thread leave its loop at the next test.  `step` = index of the step() about to run; a success
// found during launch `step` records qstep = step + 1, so runs of the same launch never see it (deterministic).
__device__ __forceinline__ bool run_done(const DState& S, int q, int step) { return S.done[q] || (S.early_exit == 2 && S.islands > 1 && S.qstep[q / S.islands] <= step) || (S.cancel && *S.cancel); }
__device__ __forceinline__ void note_success(const DState& S, int q, int steps_done)
{
    if(!S.early_exit) return;
    S.done[q] = 1;
    if(S.early_exit == 2 && S.islands > 1) atomicMin(&S.qstep[q / S.islands], steps_done);
}

// The step whose slice of the query-independent random streams (mutation table / gaussian slabs, rate exponents, fast_random values)
// run q consumes at solver step `step`.  The reference's islands are clones that replay ONE stream (SURVEY.md Q3); with
// BIOIK_OPT_ISLAND_STREAM_STRIDE island k starts k * stride steps into it, so the islands of a query diverge from their first generation.
__device__ __forceinline__ int stream_step(const DState& S, int q, int step) { return (S.islands > 1 && S.island_stride > 0) ? step + (q % S.islands) * S.island_stride : step; }

constexpr uint32_t RANDOM_BUFFER_MASK = (1u << 23) - 1;
constexpr uint32_t UNIFORM_INDEX0 = 6165936u; // XORShift64 output #1 & mask (src/ik_base.h:122)

// fast_random() values consumed by step `step` (src/ik_evolution_2.cpp:451,622): one per species
// when memetic, then one for the wipeout test.
__device__ __forceinline__ double fast_random_at(const DState& S, int step, int k)
{
    uint32_t per_step = S.memetic ? 3u : 1u;
    return S.uniform[(UNIFORM_INDEX0 + (uint32_t)step * per_step + (uint32_t)k) & RANDOM_BUFFER_MASK];
}

__device__ __forceinline__ void draw_preselect_counts(const DProblem& P, const DState& S, int q, uint32_t& rng)
{
    if(!P.has_secondary) return;
    // child_count = random_index(children.size() - population.size() - 1) + 1 + population.size()   (:369)
    for(int slot = 0; slot < 2; slot++)
        for(int g = 0; g < S.gens; g++) S.ccount[((size_t)q * 2 + slot) * S.gens + g] = (int32_t)minstd_index(rng, (uint32_t)(S.C - 3)) + 3;
}

// ---------------------------------------------------------------------------
// IKEvolution2::initialize, src/ik_evolution_2.cpp:111-230 (+ IKBase::initialize)
// ---------------------------------------------------------------------------
__global__ void k_init(const DProblem* __restrict__ Pp, DState S)
{
    const DProblem& P = *Pp;
    int q = blockIdx.x * blockDim.x + threadIdx.x;
    if(q >= S.B) return;
    const double* seed = S.seeds + (size_t)q * P.n_vars;
    const double* gp = S.goal_params + (size_t)q * P.G * GOAL_NPARAM;
    double x[MAX_GENES], vars[MAX_VARS], frames[MAX_SLOTS * 7], tips[MAX_TIPS * 7];
    for(int i = 0; i < P.n; i++) x[i] = seed[P.genes[i].var];
    // solution_fitness = computeFitness(solution)   (:129-131)
    assemble_variables(P, seed, x, vars);
    exact_fk(P, vars, frames);
    for(int t = 0; t < P.T; t++)
        for(int k = 0; k < 7; k++) tips[7 * t + k] = frames[7 * P.tip_slot[t] + k];
    S.solfit[q] = goal_fitness(P, 0, gp, tips, x, seed);
    for(int i = 0; i < P.n; i++) S.sol[(size_t)q * P.n + i] = x[i];
    for(int s = 0; s < 2; s++)
    {
        for(int k = 0; k < 2; k++)
            for(int i = 0; i < P.n; i++)
            {
                S.genes[(((size_t)q * 2 + s) * 2 + k) * P.n + i] = x[i];
                S.grads[(((size_t)q * 2 + s) * 2 + k) * P.n + i] = 0.0;
            }
        S.sfit[q * 2 + s] = 0.0; // fresh Species (SURVEY.md Q4 batch contract)
        S.impr[q * 2 + s] = 0;
    }
    uint32_t r = S.rng_seeds[q] % 2147483647u; // std::minstd_rand(seed)
    if(r == 0) r = 1;
    draw_preselect_counts(P, S, q, r);
    S.rng[q] = r;
    S.done[q] = 0;
    for(int t = 0; t < P.T; t++)
        for(int k = 0; k < 7; k++) S.carry[((size_t)q * P.T + t) * 7 + k] = k == 6 ? 1.0 : 0.0;
    S.qstep[q] = 0x7fffffff;
    S.steps[q] = 0;
    S.success[q] = 0;
}

// ---------------------------------------------------------------------------
// src/ik_evolution_2.cpp:341-346: applyConfiguration + initializeMutationApproximator
// ---------------------------------------------------------------------------
__global__ void k_prepare(const DProblem* __restrict__ Pp, DState S, int step)
{
    const DProblem& P = *Pp;
    int task = blockIdx.x * blockDim.x + threadIdx.x;
    if(task >= S.B * 2) return;
    int q = task >> 1;
    if(run_done(S, q, step)) return;
    const double* seed = S.seeds + (size_t)q * P.n_vars;
    const double* genes = S.genes + ((size_t)task * 2 + 0) * P.n;
    double vars[MAX_VARS], frames[MAX_SLOTS * 7];
    assemble_variables(P, seed, genes, vars);
    exact_fk(P, vars, frames);
    for(int t = 0; t < P.T; t++)
        for(int k = 0; k < 7; k++) S.tip0[((size_t)task * P.T + t) * 7 + k] = frames[7 * P.tip_slot[t] + k];
    for(int i = 0; i < P.n; i++) S.base[(size_t)task * P.n + i] = vars[P.genes[i].var];
    for(int t = 0; t < P.T; t++)
        for(int i = 0; i < P.n; i++)
        {
            bool masked;
            F7 d = delta_frame(P, frames, (const double*)vars, i, t, masked);
            store_frame(S.delta + (((size_t)task * P.T + t) * P.n + i) * 7, d);
        }
}

// ---------------------------------------------------------------------------
// k_evolve: one warp per task runs all generations of one step
// (src/ik_evolution_2.cpp:351-432).  Lane l owns child slots l, l+32, l+64, ...
// ---------------------------------------------------------------------------
constexpr int EVOLVE_MAX_CPL = 8; // children per lane => population <= 256

struct EvolveSmem // per-warp shared-memory carve-up, in doubles
{
    int n, T, G;
    __host__ __device__ int off_delta() const { return 0; }
    __host__ __device__ int off_tip0() const { return off_delta() + T * n * 7; }
    __host__ __device__ int off_base() const { return off_tip0() + T * 7; }
    __host__ __device__ int off_g0() const { return off_base() + n; }  // individuals[0].genes
    __host__ __device__ int off_g1() const { return off_g0() + n; }    // individuals[1].genes
    __host__ __device__ int off_gr0() const { return off_g1() + n; }   // individuals[0].gradients
    __host__ __device__ int off_gr1() const { return off_gr0() + n; }  // individuals[1].gradients
    __host__ __device__ int off_gp() const { return off_gr1() + n; }   // goal params
    __host__ __device__ int off_sf() const { return off_gp() + G * GOAL_NPARAM; } // secondary fitness per child slot (256)
    __host__ __device__ int total() const { return off_sf() + 256; }
};

__device__ __forceinline__ uint64_t fitness_key(double f)
{
    // fitness is a sum of weighted squares: >= +0, so the IEEE bit pattern orders like the value.
    // NaN never wins a `f < fmin` test (:422): give it the largest key.
    return (f != f) ? 0xFFFFFFFFFFFFFFFFull : (uint64_t)__double_as_longlong(f);
}

// warp-wide argmin of (key, pos); ties -> lowest pos (strict `<` scan in position order, :419-423)
__device__ __forceinline__ void warp_argmin(uint64_t& key, int& pos, int& child)
{
#pragma unroll
    for(int o = 16; o > 0; o >>= 1)
    {
        uint64_t k2 = __shfl_xor_sync(0xffffffffu, key, o);
        int p2 = __shfl_xor_sync(0xffffffffu, pos, o);
        int c2 = __shfl_xor_sync(0xffffffffu, child, o);
        if(k2 < key || (k2 == key && p2 < pos))
        {
            key = k2;
            pos = p2;
            child = c2;
        }
    }
}

__global__ void __launch_bounds__(128) k_evolve(const DProblem* __restrict__ Pp, DState S, int step)
{
    extern __shared__ double smem[];
    const DProblem& P = *Pp;
    const int lane = threadIdx.x & 31;
    const int warp_in_block = threadIdx.x >> 5;
    const int task = blockIdx.x * (blockDim.x >> 5) + warp_in_block;
    if(task >= S.B * 2) return;
    const int q = task >> 1, slot = task & 1;
    if(run_done(S, q, step)) return;
    const int n = P.n, T = P.T, C = S.C;
    EvolveSmem L{n, T, P.G};
    double* W = smem + (size_t)warp_in_block * L.total();
    double *s_delta = W + L.off_delta(), *s_tip0 = W + L.off_tip0(), *s_base = W + L.off_base();
    double *s_g0 = W + L.off_g0(), *s_g1 = W + L.off_g1(), *s_gr0 = W + L.off_gr0(), *s_gr1 = W + L.off_gr1();
    double *s_gp = W + L.off_gp(), *s_sf = W + L.off_sf();
    const double* seed = S.seeds + (size_t)q * P.n_vars;

    // stage the task's approximator, parents and goal parameters (coalesced)
    for(int i = lane; i < T * n * 7; i += 32) s_delta[i] = S.delta[(size_t)task * T * n * 7 + i];
    for(int i = lane; i < T * 7; i += 32) s_tip0[i] = S.tip0[(size_t)task * T * 7 + i];
    for(int i = lane; i < n; i += 32)
    {
        s_base[i] = S.base[(size_t)task * n + i];
        s_g0[i] = S.genes[((size_t)task * 2 + 0) * n + i];
        s_g1[i] = S.genes[((size_t)task * 2 + 1) * n + i];
        s_gr0[i] = S.grads[((size_t)task * 2 + 0) * n + i];
        s_gr1[i] = S.grads[((size_t)task * 2 + 1) * n + i];
    }
    for(int i = lane; i < P.G * GOAL_NPARAM; i += 32) s_gp[i] = S.goal_params[(size_t)q * P.G * GOAL_NPARAM + i];
    __syncwarp();

    const int stride4 = (n + 3) / 4 * 4; // rr += (gene_count + 3) / 4 * 4   (:301)
    double x[MAX_GENES], cg[MAX_GENES], F[MAX_TIPS * 7];

    for(int gen = 0; gen < S.gens; gen++)
    {
        const int call = (stream_step(S, q, step) * 2 + slot) * S.gens + gen;
        const double* rr_base = S.gauss + S.gauss_off[call];
        const uint8_t* rexp = S.rate_exp + (size_t)call * (C - 2);
        const int child_count = P.has_secondary ? S.ccount[((size_t)q * 2 + slot) * S.gens + gen] : C;

        double fit[EVOLVE_MAX_CPL];
        int posn[EVOLVE_MAX_CPL];

        // pre-selection by secondary objectives (:366-378): position = 2 + stable rank of the secondary fitness
        if(P.has_secondary)
        {
            for(int k = 0; k < EVOLVE_MAX_CPL; k++)
            {
                int c = lane + 32 * k;
                if(c >= 2 && c < C)
                {
                    reproduce_child(P, c, rexp[c - 2], rr_base + (size_t)(c - 2) * stride4, s_g0, s_gr0, s_gr1, x, nullptr);
                    s_sf[c] = goal_fitness(P, 1, s_gp, nullptr, x, seed);
                }
            }
            __syncwarp();
        }
#pragma unroll
        for(int k = 0; k < EVOLVE_MAX_CPL; k++)
        {
            int c = lane + 32 * k;
            fit[k] = 0.0;
            posn[k] = 0x7fffffff;
            if(c >= C) continue;
            int pos = c;
            if(P.has_secondary && c >= 2)
            {
                double mine = s_sf[c];
                int rank = 0;
                for(int o = 2; o < C; o++)
                {
                    double other = s_sf[o];
                    rank += (other < mine || (other == mine && o < c)) ? 1 : 0;
                }
                pos = 2 + rank;
            }
            if(pos >= child_count) continue; // not evaluated, not eligible (:394-406,:412-414)
            const double* gsrc;
            if(c == 0) gsrc = s_g0;       // keep parents (:381-388)
            else if(c == 1) gsrc = s_g1;
            else
            {
                reproduce_child(P, c, rexp[c - 2], rr_base + (size_t)(c - 2) * stride4, s_g0, s_gr0, s_gr1, x, nullptr);
                gsrc = x;
            }
            approx_frames(T, n, s_tip0, s_delta, s_base, gsrc, F); // genotype-phenotype mapping (:391-398)
            fit[k] = goal_fitness(P, 0, s_gp, F, gsrc, seed);     // fitness (:401-407)
            posn[k] = pos;
        }

        // selection (:410-431): two passes of a strict-< scan in position order
        uint64_t key = 0xFFFFFFFFFFFFFFFFull;
        int bpos = 0x7fffffff, bchild = -1;
#pragma unroll
        for(int k = 0; k < EVOLVE_MAX_CPL; k++)
        {
            uint64_t kk = fitness_key(fit[k]);
            if(posn[k] != 0x7fffffff && (kk < key || (kk == key && posn[k] < bpos)))
            {
                key = kk;
                bpos = posn[k];
                bchild = lane + 32 * k;
            }
        }
        warp_argmin(key, bpos, bchild);
        // position 0 holds parent 0 (lane 0, k = 0): if its fitness is NaN nothing beats it (:418-422)
        double f_pos0 = __shfl_sync(0xffffffffu, fit[0], 0);
        double f_pos1 = __shfl_sync(0xffffffffu, fit[0], 1);
        int w1_pos = bpos, w1_child = bchild;
        if(f_pos0 != f_pos0) { w1_pos = 0; w1_child = 0; }
        // second pass: everything except winner 1; after the swap (:424) the element that was at
        // position 0 sits at position w1_pos
        key = 0xFFFFFFFFFFFFFFFFull;
        bpos = 0x7fffffff;
        bchild = -1;
#pragma unroll
        for(int k = 0; k < EVOLVE_MAX_CPL; k++)
        {
            int c = lane + 32 * k;
            if(posn[k] == 0x7fffffff || c == w1_child) continue;
            int p = (posn[k] == 0) ? w1_pos : posn[k];
            uint64_t kk = fitness_key(fit[k]);
            if(kk < key || (kk == key && p < bpos))
            {
                key = kk;
                bpos = p;
                bchild = c;
            }
        }
        warp_argmin(key, bpos, bchild);
        int w2_child = bchild;
        {
            // the scan starts at position 1: its occupant wins if its fitness is NaN
            int occ1_child = (w1_pos == 1) ? 0 : 1; // occupant of position 1 after the first swap
            double f_occ1 = (occ1_child == 0) ? f_pos0 : f_pos1;
            if(f_occ1 != f_occ1) w2_child = occ1_child;
        }

        // materialise the winners from the OLD parents, then overwrite the parents (:426-430)
        bool is_w = (lane == 0) || (lane == 1);
        int wc = (lane == 0) ? w1_child : w2_child;
        if(is_w)
        {
            if(wc == 0)
                for(int i = 0; i < n; i++) { x[i] = s_g0[i]; cg[i] = s_gr0[i]; }
            else if(wc == 1)
                for(int i = 0; i < n; i++) { x[i] = s_g1[i]; cg[i] = s_gr1[i]; }
            else
                reproduce_child(P, wc, rexp[wc - 2], rr_base + (size_t)(wc - 2) * stride4, s_g0, s_gr0, s_gr1, x, cg);
        }
        __syncwarp();
        if(lane == 0)
            for(int i = 0; i < n; i++) { s_g0[i] = x[i]; s_gr0[i] = cg[i]; }
        if(lane == 1)
            for(int i = 0; i < n; i++) { s_g1[i] = x[i]; s_gr1[i] = cg[i]; }
        __syncwarp();
    }

    for(int i = lane; i < n; i += 32)
    {
        S.genes[((size_t)task * 2 + 0) * n + i] = s_g0[i];
        S.genes[((size_t)task * 2 + 1) * n + i] = s_g1[i];
        S.grads[((size_t)task * 2 + 0) * n + i] = s_gr0[i];
        S.grads[((size_t)task * 2 + 1) * n + i] = s_gr1[i];
    }
}

// ---------------------------------------------------------------------------
// memetic optimisation of individuals[0], src/ik_evolution_2.cpp:436-570
// ---------------------------------------------------------------------------
__global__ void k_memetic(const DProblem* __restrict__ Pp, DState S, int step)
{
    const DProblem& P = *Pp;
    int task = blockIdx.x * blockDim.x + threadIdx.x;
    if(task >= S.B * 2) return;
    const int q = task >> 1, slot = task & 1;
    if(run_done(S, q, step)) return;
    const int n = P.n, T = P.T;
    const double* seed = S.seeds + (size_t)q * P.n_vars;
    const double* gp = S.goal_params + (size_t)q * P.G * GOAL_NPARAM;
    const double* delta = S.delta + (size_t)task * T * n * 7;
    const double* tip0 = S.tip0 + (size_t)task * T * 7;
    const double* base = S.base + (size_t)task * n;
    double* genes = S.genes + ((size_t)task * 2 + 0) * n; // individual = population[0]

    double ind[MAX_GENES], temp[MAX_GENES], grad[MAX_GENES], ph2[MAX_TIPS * 7], ph3[MAX_TIPS * 7];
    for(int i = 0; i < n; i++) ind[i] = genes[i];

    double dp = 0.0000001; // :450
    if(fast_random_at(S, stream_step(S, q, step), slot) < 0.5) dp = -dp; // :451
    bool changed = false;
    for(int generation = 0; generation < S.memetic_iters; generation++)
    {
        for(int i = 0; i < n; i++) temp[i] = ind[i]; // :460
        approx_frames(T, n, tip0, delta, base, temp, ph2); // :462
        double f2p = goal_fitness(P, 0, gp, ph2, temp, seed);                                   // :463
        double fa = f2p + (P.has_secondary ? goal_fitness(P, 1, gp, nullptr, temp, seed) : 0.0); // :464  (empty sum = 0.0)
        for(int i = 0; i < n; i++) // :465-474
        {
            temp[i] = ind[i] + dp;
            approx_frames1(T, n, delta, i, dp, ph2, ph3);
            double fb = 0.0; // computeCombinedFitnessActiveVariables, src/ik_base.h:179-185
            fb += goal_fitness(P, 0, gp, ph3, temp, seed);
            fb += P.has_secondary ? goal_fitness(P, 1, gp, nullptr, temp, seed) : 0.0;
            temp[i] = ind[i];
            grad[i] = fb - fa;
        }
        double sum = dp * dp; // :477-482
        for(int i = 0; i < n; i++) sum += fabs(grad[i]);
        double f = 1.0 / sum * dp;
        for(int i = 0; i < n; i++) grad[i] *= f;

        for(int i = 0; i < n; i++) temp[i] = ind[i] - grad[i]; // :485-488
        approx_frames(T, n, tip0, delta, base, temp, ph3);
        double f1 = 0.0;
        f1 += goal_fitness(P, 0, gp, ph3, temp, seed);
        f1 += P.has_secondary ? goal_fitness(P, 1, gp, nullptr, temp, seed) : 0.0;
        double f2 = fa;
        for(int i = 0; i < n; i++) temp[i] = ind[i] + grad[i]; // :492-495
        approx_frames(T, n, tip0, delta, base, temp, ph3);
        double f3 = 0.0;
        f3 += goal_fitness(P, 0, gp, ph3, temp, seed);
        f3 += P.has_secondary ? goal_fitness(P, 1, gp, nullptr, temp, seed) : 0.0;

        if(S.memetic == 'q') // :498-542
        {
            double v1 = (f2 - f1);
            double v2 = (f3 - f2);
            double v = (v1 + v2) * 0.5;
            double a = (v1 - v2);
            double step_size = v / a;
            for(int i = 0; i < n; i++) temp[i] = clampd(ind[i] + grad[i] * step_size * 1.0, P.genes[i].clip_min, P.genes[i].clip_max); // :525
        }
        else // 'l', :545-568
        {
            double cost_diff = (f3 - f1) * 0.5;
            double step_size = f2 / cost_diff;
            for(int i = 0; i < n; i++) temp[i] = clampd(ind[i] - grad[i] * step_size, P.genes[i].clip_min, P.genes[i].clip_max); // :554
        }
        approx_frames(T, n, tip0, delta, base, temp, ph2);
        double f4p = goal_fitness(P, 0, gp, ph2, temp, seed);
        if(f4p < f2p) // :530-538 / :559-567
        {
            for(int i = 0; i < n; i++) ind[i] = temp[i];
            changed = true;
            continue;
        }
        else
            break;
    }
    if(changed)
        for(int i = 0; i < n; i++) genes[i] = ind[i];
}

// ---------------------------------------------------------------------------
// species block (src/ik_evolution_2.cpp:604-645) + driver check (src/ik_parallel.h:173-181)
// ---------------------------------------------------------------------------
__device__ __forceinline__ double exact_primary_fitness(const DProblem& P, const double* seed, const double* gp, const double* genes, double* tips_out)
{
    double vars[MAX_VARS], frames[MAX_SLOTS * 7];
    assemble_variables(P, seed, genes, vars);
    exact_fk(P, vars, frames);
    for(int t = 0; t < P.T; t++)
        for(int k = 0; k < 7; k++) tips_out[7 * t + k] = frames[7 * P.tip_slot[t] + k];
    return goal_fitness(P, 0, gp, tips_out, genes, seed);
}

__global__ void k_species(const DProblem* __restrict__ Pp, DState S, int step)
{
    const DProblem& P = *Pp;
    int q = blockIdx.x * blockDim.x + threadIdx.x;
    if(q >= S.B) return;
    if(run_done(S, q, step)) return;
    const int n = P.n;
    const double* seed = S.seeds + (size_t)q * P.n_vars;
    const double* gp = S.goal_params + (size_t)q * P.G * GOAL_NPARAM;
    double tips[MAX_TIPS * 7];
    double* G0 = S.genes + ((size_t)q * 2 + 0) * 2 * n; // species slot 0: [2 individuals][n]
    double* G1 = S.genes + ((size_t)q * 2 + 1) * 2 * n;
    double* R0 = S.grads + ((size_t)q * 2 + 0) * 2 * n;
    double* R1 = S.grads + ((size_t)q * 2 + 1) * 2 * n;

    // :608-614
    double f0 = exact_primary_fitness(P, seed, gp, G0, tips);
    double f1 = exact_primary_fitness(P, seed, gp, G1, tips);
    int i0 = (f0 != S.sfit[q * 2 + 0]), i1 = (f1 != S.sfit[q * 2 + 1]);
    // :617 sort ascending (2 elements: swap iff species[1] < species[0])
    if(f1 < f0)
    {
        for(int i = 0; i < 2 * n; i++)
        {
            double a = G0[i]; G0[i] = G1[i]; G1[i] = a;
            double b = R0[i]; R0[i] = R1[i]; R1[i] = b;
        }
        double tf = f0; f0 = f1; f1 = tf;
        int ti = i0; i0 = i1; i1 = ti;
    }
    S.sfit[q * 2 + 0] = f0; S.sfit[q * 2 + 1] = f1;
    S.impr[q * 2 + 0] = i0; S.impr[q * 2 + 1] = i1;
    // :620-637 wipeout of species[1]
    uint32_t rng = S.rng[q];
    double u = fast_random_at(S, stream_step(S, q, step), S.memetic ? 2 : 0);
    if(u < 0.1 || !i1)
    {
        for(int i = 0; i < n; i++)
        {
            double g = minstd_random(rng, P.genes[i].vmin, P.genes[i].vmax); // :629 (getMin/getMax, unclipped)
            G1[i] = g;
            G1[n + i] = g; // individuals[i] = individuals[0]
            R1[i] = 0.0;
            R1[n + i] = 0.0;
        }
    }
    // :640-644
    if(f0 < S.solfit[q])
    {
        for(int i = 0; i < n; i++) S.sol[(size_t)q * n + i] = G0[i];
        S.solfit[q] = f0;
    }
    int steps = S.steps[q] + 1;
    S.steps[q] = steps;
    // driver: step() x4 then test (src/ik_parallel.h:165-181); with a step budget the last burst may be short
    if((steps % 4) == 0 || steps == S.total_steps)
    {
        const double* sol = S.sol + (size_t)q * n;
        exact_primary_fitness(P, seed, gp, sol, tips);
        int ok = check_solution(P, gp, tips, sol, seed) ? 1 : 0;
        S.success[q] = ok;
        if(ok) note_success(S, q, steps);
    }
    draw_preselect_counts(P, S, q, rng); // random_index draws of the NEXT step's generations (:369)
    S.rng[q] = rng;
}

// outputs: getSolution() (full variable vector), its primary fitness (src/ik_parallel.h:181), success
__global__ void k_finalize(const DProblem* __restrict__ Pp, DState S, double* out_solutions, double* out_fitness, int32_t* out_success, int32_t* out_steps)
{
    const DProblem& P = *Pp;
    int q = blockIdx.x * blockDim.x + threadIdx.x;
    if(q >= S.B) return;
    const double* seed = S.seeds + (size_t)q * P.n_vars;
    const double* gp = S.goal_params + (size_t)q * P.G * GOAL_NPARAM;
    const double* sol = S.sol + (size_t)q * P.n;
    double tips[MAX_TIPS * 7];
    double f = exact_primary_fitness(P, seed, gp, sol, tips);
    if(out_solutions)
        for(int v = 0; v < P.n_vars; v++)
        {
            int g = P.gene_of_var[v];
            out_solutions[(size_t)q * P.n_vars + v] = g >= 0 ? sol[g] : seed[v];
        }
    if(out_fitness) out_fitness[q] = f;
    if(out_success) out_success[q] = check_solution(P, gp, tips, sol, seed) ? 1 : 0;
    if(out_steps) out_steps[q] = S.steps[q];
}

// ---------------------------------------------------------------------------
// Many differently seeded islands of ONE query (SURVEY.md §8(f) rows 1 and 3): the batch holds Q x islands runs,
// run q * islands + k being island k of query q.
// ---------------------------------------------------------------------------
#ifndef BIOIK_HOSTSIM
// host polling between 4-step bursts: *count = number of runs that would still execute step `step`
__global__ void k_count_active(DState S, int step, int32_t* count)
{
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    const bool on = q < S.B && !run_done(S, q, step);
    const unsigned m = __ballot_sync(0xffffffffu, on);
    if((threadIdx.x & 31) == 0 && m) atomicAdd(count, __popc(m));
}
#endif

// island inputs from query inputs: goal parameters [Q][G][NPARAM] and seeds [Q][n_vars] repeated `islands` times
__global__ void k_expand_islands(int Q, int islands, int per_gp, int per_seed, const double* gp, const double* seeds, double* gp_out, double* seeds_out)
{
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t ngp = gp ? (size_t)Q * islands * per_gp : 0, nsd = (size_t)Q * islands * per_seed;
    if(idx < ngp)
    {
        const size_t b = idx / per_gp, k = idx - b * per_gp;
        gp_out[idx] = gp[(b / islands) * per_gp + k];
    }
    if(idx < nsd)
    {
        const size_t b = idx / per_seed, k = idx - b * per_seed;
        seeds_out[idx] = seeds[(b / islands) * per_seed + k];
    }
}

// IKParallel::solve's selection among its threads (src/ik_parallel.h:218-258) + the plugin's angle wrap
// (src/kinematics_plugin.cpp:580-611) for query q; inputs are the per-run outputs of k_finalize.
__global__ void k_select_islands(const DProblem* __restrict__ Pp, int Q, int islands, const double* goal_params, const double* seeds, const double* sol, const double* fit, const int32_t* succ, const int32_t* steps, int wrap,
                                 double* out_solutions, double* out_fitness, int32_t* out_success, int32_t* out_island, int32_t* out_steps)
{
    const DProblem& P = *Pp;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if(q >= Q) return;
    const size_t b0 = (size_t)q * islands;
    const double* seed = seeds + b0 * P.n_vars;       // every island of the query has the query's seed
    const double* gp = goal_params + b0 * P.G * GOAL_NPARAM;
    double best;
    const int k = select_island(P, islands, gp, seed, sol + b0 * P.n_vars, fit + b0, succ + b0, &best);
    const double* s = sol + (b0 + k) * P.n_vars;
    for(int v = 0; v < P.n_vars; v++)
    {
        double x = s[v];
        const int g = P.gene_of_var[v];
        if(wrap && g >= 0 && P.wrap_gene[g]) x = wrap_angle(x, seed[v], P.genes[g].vmin, P.genes[g].vmax);
        out_solutions[(size_t)q * P.n_vars + v] = x;
    }
    if(out_fitness) out_fitness[q] = best;
    if(out_success) out_success[q] = succ[b0 + k];
    if(out_island) out_island[q] = k;
    if(out_steps) out_steps[q] = steps[b0 + k];
}

// ---------------------------------------------------------------------------
// component kernels (parity tests of the individual rows of SURVEY.md §8(a))
// ---------------------------------------------------------------------------
__global__ void k_fk_batch(const DProblem* __restrict__ Pp, int B, const double* variables, double* out_tips)
{
    const DProblem& P = *Pp;
    int b = blockIdx.x * blockDim.x + threadIdx.x;
    if(b >= B) return;
    double vars[MAX_VARS], frames[MAX_SLOTS * 7];
    for(int v = 0; v < P.n_vars; v++) vars[v] = variables[(size_t)b * P.n_vars + v];
    for(int m = 0; m < P.n_mimic; m++) vars[P.mimics[m].dest] = vars[P.mimics[m].src] * P.mimics[m].factor + P.mimics[m].offset;
    exact_fk(P, vars, frames);
    for(int t = 0; t < P.T; t++)
        for(int k = 0; k < 7; k++) out_tips[((size_t)b * P.T + t) * 7 + k] = frames[7 * P.tip_slot[t] + k];
}

__global__ void k_approx_batch(const DProblem* __restrict__ Pp, int B, const double* variables, double* out_delta)
{
    const DProblem& P = *Pp;
    int b = blockIdx.x * blockDim.x + threadIdx.x;
    if(b >= B) return;
    double vars[MAX_VARS], frames[MAX_SLOTS * 7];
    for(int v = 0; v < P.n_vars; v++) vars[v] = variables[(size_t)b * P.n_vars + v];
    for(int m = 0; m < P.n_mimic; m++) vars[P.mimics[m].dest] = vars[P.mimics[m].src] * P.mimics[m].factor + P.mimics[m].offset;
    exact_fk(P, vars, frames);
    for(int t = 0; t < P.T; t++)
        for(int i = 0; i < P.n; i++)
        {
            bool masked;
            F7 d = delta_frame(P, frames, (const double*)vars, i, t, masked);
            store_frame(out_delta + (((size_t)b * P.T + t) * P.n + i) * 7, d);
        }
}

__global__ void k_approx_fitness(const DProblem* __restrict__ Pp, int B, int M, const double* goal_params, const double* seeds, const double* base_variables, const double* genotypes, double* out_primary, double* out_secondary,
                                 double* scratch_delta)
{
    const DProblem& P = *Pp;
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if(idx >= B * M) return;
    int b = idx / M;
    const int n = P.n, T = P.T;
    double vars[MAX_VARS], frames[MAX_SLOTS * 7], tip0[MAX_TIPS * 7], base[MAX_GENES], F[MAX_TIPS * 7];
    for(int v = 0; v < P.n_vars; v++) vars[v] = base_variables[(size_t)b * P.n_vars + v];
    for(int m = 0; m < P.n_mimic; m++) vars[P.mimics[m].dest] = vars[P.mimics[m].src] * P.mimics[m].factor + P.mimics[m].offset;
    exact_fk(P, vars, frames);
    double* delta = scratch_delta + (size_t)idx * T * n * 7;
    for(int t = 0; t < T; t++)
    {
        for(int k = 0; k < 7; k++) tip0[7 * t + k] = frames[7 * P.tip_slot[t] + k];
        for(int i = 0; i < n; i++)
        {
            bool masked;
            store_frame(delta + ((size_t)t * n + i) * 7, delta_frame(P, frames, (const double*)vars, i, t, masked));
        }
    }
    for(int i = 0; i < n; i++) base[i] = vars[P.genes[i].var];
    const double* x = genotypes + (size_t)idx * n;
    const double* gp = goal_params + (size_t)b * P.G * GOAL_NPARAM;
    const double* seed = seeds + (size_t)b * P.n_vars;
    approx_frames(T, n, tip0, delta, base, x, F);
    if(out_primary) out_primary[idx] = goal_fitness(P, 0, gp, F, x, seed);
    if(out_secondary) out_secondary[idx] = goal_fitness(P, 1, gp, nullptr, x, seed);
}

} // namespace bioik

#include "bioik_evolve_fast.cuh"
#include "bioik_serial.cuh"
#include "bioik_memetic_group.cuh"
#include "bioik_persist.cuh"
