// bioik_serial.cuh — the fused per-task "serial" kernel: everything of step() that is one
// dependent chain per species (DESIGN.md §6):
//   MEMETIC  quadratic / linear line search on individuals[0]           src/ik_evolution_2.cpp:436-570
//   SPECIES  exact fitness, species sort, wipeout, solution update      src/ik_evolution_2.cpp:604-645
//            + the driver's success test                                src/ik_parallel.h:173-181
//   PREPARE  exact FK + Jacobian + delta frames for the next step       src/ik_evolution_2.cpp:341-346
// One thread per task (query, species slot); the two species of a query sit in adjacent lanes and
// meet through warp shuffles in the species block.  All per-thread arrays are shared-memory COLUMNS
// (element e of thread t at base[e * blockDim.x + t]: conflict-free), the flattened problem sits in
// the constant bank (kernel parameter), so the dependent chains never wait on local or global memory.
// The exact FK of the species block is reused by PREPARE unless the species was wiped out.
#pragma once

#include "bioik_dev.cuh"
#include "bioik_evolve_fast.cuh" // link_goal_value

#ifdef BIOIK_HOSTSIM
#define BIOIK_PROBLEM_PARAM const DProblem& P
#else
#define BIOIK_PROBLEM_PARAM const __grid_constant__ DProblem P
#endif

namespace bioik
{

enum SerialPhase { PH_MEMETIC = 1, PH_SPECIES = 2, PH_PREPARE = 4 };

// host-computed launch plan: which per-thread arrays fit in shared memory at which block size
struct SerialPlan
{
    int block;       // threads per block
    int delta_smem;  // delta frames [T][n][7] in shared memory (else read from the HBM state, L1/L2 cached)
    int frames_smem; // link frames [L][7] in shared memory (else thread-local memory)
    int per_thread;  // doubles per thread
    size_t smem_bytes;
};

__host__ __device__ inline int serial_fixed_doubles(const DProblem& P) { return 4 * P.n /*ind,temp,grad,stash*/ + 3 * 7 * P.T /*ph2,ph3,tip0*/ + P.n /*base*/ + GOAL_NPARAM * P.G + P.n_vars; }

// The kernel is latency-bound (one dependent chain per thread), so what matters is that ALL tasks are
// resident at once (a second wave doubles the time): blocks of one warp pack best; pick the most
// on-chip variant whose resident threads per SM cover ceil(tasks / SMs).
inline SerialPlan make_serial_plan(const DProblem& P, int tasks = 0, int sm_count = 132, size_t smem_per_sm = 227 * 1024)
{
    const int fixed = serial_fixed_doubles(P), dl = 7 * P.T * P.n, fr = 7 * P.L;
    const int need = tasks > 0 ? (tasks + sm_count - 1) / sm_count : 64; // threads per SM for a single wave
    SerialPlan best;
    int best_resident = -1;
    const int variants[4][2] = {{1, 1}, {1, 0}, {0, 1}, {0, 0}}; // {delta on chip, frames on chip}
    for(int v = 0; v < 4; v++)
    {
        SerialPlan pl;
        pl.block = 32;
        pl.delta_smem = variants[v][0];
        pl.frames_smem = variants[v][1];
        pl.per_thread = fixed + (pl.delta_smem ? dl : 0) + (pl.frames_smem ? fr : 0);
        pl.smem_bytes = (size_t)pl.per_thread * pl.block * sizeof(double);
        if(pl.smem_bytes + 1024 > smem_per_sm) continue;
        int blocks = (int)(smem_per_sm / (pl.smem_bytes + 1024)); // 1 KB reserved per resident block
        if(blocks > 32) blocks = 32;
        const int resident = blocks * pl.block;
        if(resident >= need) return pl; // most on-chip variant that still runs in one wave
        if(resident > best_resident)
        {
            best_resident = resident;
            best = pl;
        }
    }
    return best;
}

// problems for which k_serial carries the unrolled register-resident memetic step (memetic_single_pose): one primary
// PoseGoal, one tip, 6 or 7 genes that all move the tip (the MoveIt plugin's default problem on a 6/7-DOF arm)
__host__ __device__ inline bool has_unrolled_memetic(const DProblem& P)
{
    bool ok = (P.G == 1 && P.T == 1 && P.goals[0].type == G_POSE && !P.goals[0].secondary) && (P.n == 6 || P.n == 7);
    for(int i = 0; ok && i < P.n; i++) ok = (P.genes[i].tipmask & 1) != 0;
    return ok;
}

// asynchronous 8-byte global -> shared copies (LDGSTS): a thread queues every input of its task back to back and waits
// once, instead of paying one memory round trip per load-store pair of a staging loop
BIOIK_HD void stage8(double* dst_shared, const double* src_global)
{
#ifdef BIOIK_HOSTSIM
    *dst_shared = *src_global;
#else
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst_shared);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(src_global) : "memory");
#endif
}
BIOIK_HD void stage_wait()
{
#ifndef BIOIK_HOSTSIM
    asm volatile("cp.async.wait_all;" ::: "memory");
#endif
}

// assemble_variables when the non-gene entries of `vars` already hold the seed: gene entries, then updateMimic
template <class AG, class AV> BIOIK_HD void assemble_genes(const DProblem& P, AG genes, AV vars)
{
    for(int i = 0; i < P.n; i++) vars[P.genes[i].var] = genes[i];
    for(int m = 0; m < P.n_mimic; m++) vars[P.mimics[m].dest] = vars[P.mimics[m].src] * P.mimics[m].factor + P.mimics[m].offset;
}

template <class AF, class AT> BIOIK_HD void copy_tips(const DProblem& P, AF frames, AT tips)
{
    for(int t = 0; t < P.T; t++)
        for(int k = 0; k < 7; k++) tips[7 * t + k] = frames[7 * P.tip_slot[t] + k];
}

// The memetic line search (src/ik_evolution_2.cpp:436-570) for the plugin's default problem - exactly one primary
// PoseGoal on one tip, every gene moving that tip - with the gene count as a compile-time constant: genes, gradient,
// base point, frames and goal parameters live in registers and every loop is unrolled, so the n gradient probes, the
// two support points and the seven frame components are independent instruction streams the scheduler can overlap
// (the thread-per-task kernel has about one warp per scheduler, so it lives on instruction-level parallelism).
// Same operations in the same order as the general loop of k_serial.  Returns nothing; `ind` is updated in place.
template <int NS, class IndCol, class DeltaColT, class TipCol, class BaseCol, class GpCol>
BIOIK_HD void memetic_single_pose(const DProblem& P, const DState& S, IndCol ind, DeltaColT delta, TipCol tip0, BaseCol base, GpCol gp, double dp, bool quad)
{
    double pg[8], t0r[7], x[NS], bs[NS], gr[NS], tm[NS], cmin[NS], cmax[NS];
#pragma unroll
    for(int k = 0; k < 8; k++) pg[k] = gp[k];
#pragma unroll
    for(int k = 0; k < 7; k++) t0r[k] = tip0[k];
#pragma unroll
    for(int i = 0; i < NS; i++) x[i] = ind[i], bs[i] = base[i], cmin[i] = P.genes[i].clip_min, cmax[i] = P.genes[i].clip_max;
    const double wsq = P.goals[0].weight_sq;
    auto full_frames = [&](const double (&g)[NS], double (&F)[7]) {
#pragma unroll
        for(int k = 0; k < 7; k++) F[k] = t0r[k];
#pragma unroll
        for(int i = 0; i < NS; i++)
        {
            const double d = g[i] - bs[i]; // :1086
            const DeltaColT D = delta + 7 * i;
#pragma unroll
            for(int k = 0; k < 7; k++) F[k] = BIOIK_FMA(d, D[k], F[k]);
        }
    };
    auto pose = [&](const double (&F)[7]) { return 0.0 + link_goal_value(G_POSE, pg, F) * wsq; }; // sum = 0.0; sum += e * weight_sq
    for(int generation = 0; generation < S.memetic_iters; generation++)
    {
        double F2[7];
        full_frames(x, F2);          // :460-462
        const double f2p = pose(F2); // :463
        const double fa = f2p + 0.0; // :464 (no secondary goals)
#pragma unroll
        for(int i = 0; i < NS; i++) // :465-474
        {
            double F3[7];
            const DeltaColT D = delta + 7 * i;
#pragma unroll
            for(int k = 0; k < 7; k++) F3[k] = BIOIK_FMA(dp, D[k], F2[k]); // :469
            double fb = 0.0;
            fb += pose(F3);
            fb += 0.0;
            gr[i] = fb - fa;
        }
        double sum = dp * dp; // :477-482
#pragma unroll
        for(int i = 0; i < NS; i++) sum += BIOIK_FABS(gr[i]);
        const double f = 1.0 / sum * dp;
#pragma unroll
        for(int i = 0; i < NS; i++) gr[i] *= f;
        double FA[7], FB[7];
#pragma unroll
        for(int i = 0; i < NS; i++) tm[i] = x[i] - gr[i]; // :485-488
        full_frames(tm, FA);
        double f1 = 0.0;
        f1 += pose(FA);
        f1 += 0.0;
        const double f2 = fa;
#pragma unroll
        for(int i = 0; i < NS; i++) tm[i] = x[i] + gr[i]; // :492-495
        full_frames(tm, FB);
        double f3 = 0.0;
        f3 += pose(FB);
        f3 += 0.0;
        if(quad) // :502-506,:525
        {
            double v1 = (f2 - f1);
            double v2 = (f3 - f2);
            double v = (v1 + v2) * 0.5;
            double a = (v1 - v2);
            double step_size = v / a;
#pragma unroll
            for(int i = 0; i < NS; i++) tm[i] = clampd(x[i] + gr[i] * step_size * 1.0, cmin[i], cmax[i]);
        }
        else // :549-554
        {
            double cost_diff = (f3 - f1) * 0.5;
            double step_size = f2 / cost_diff;
#pragma unroll
            for(int i = 0; i < NS; i++) tm[i] = clampd(x[i] - gr[i] * step_size, cmin[i], cmax[i]);
        }
        full_frames(tm, F2); // :526 / :555
        const double f4p = pose(F2);
        if(f4p < f2p) // :530-538 / :559-567
        {
#pragma unroll
            for(int i = 0; i < NS; i++) x[i] = tm[i];
            continue;
        }
        else
            break;
    }
#pragma unroll
    for(int i = 0; i < NS; i++) ind[i] = x[i];
}

// BS = threads per block (column stride), DS = delta frames in shared memory, FS = link frames in shared memory
// The serial work of BS tasks, one thread each (tid = the thread's column in `smem`, task_raw = its task).  Called by k_serial
// (one block of BS threads per call) and by the persistent solve kernel (bioik_persist.cuh: one warp, BS = 32).
template <int BS, bool DS, bool FS> __device__ __forceinline__ void serial_tasks(const DProblem& P, const DState& S, int step, int phases, double* smem, int tid, int task_raw)
{
    typedef FixedCol<double, BS> SC;         // shared-memory column
    typedef FixedCol<const double, BS> CSC;
    typedef FixedCol<double, 1> GC;          // plain array (global / local)
    typedef typename std::conditional<DS, SC, GC>::type DeltaCol;
    typedef typename std::conditional<FS, SC, GC>::type FrameCol;

    const bool valid = task_raw < 2 * S.B;
    const int task = valid ? task_raw : 2 * S.B - 1;
    const int q = task >> 1, slot = task & 1;
    const bool active = valid && !run_done(S, q, step);
    const int n = P.n, T = P.T, G = P.G;

    // ---- per-thread columns --------------------------------------------------------------------
    int off = 0;
    auto col = [&](int len) {
        SC c{smem + off * BS + tid};
        off += len;
        return c;
    };
    const SC ind = col(n), temp = col(n), grad = col(n), stash = col(n), ph2 = col(7 * T), ph3 = col(7 * T), tip0 = col(7 * T), base = col(n), gp = col(GOAL_NPARAM * G), vars = col(P.n_vars);
    DeltaCol delta;
    if(DS)
        delta.p = smem + off * BS + tid, off += 7 * T * n;
    else
        delta.p = S.delta + (size_t)task * T * n * 7;
    double lf[FS ? 1 : MAX_SLOTS * 7]; // link frames in thread-local memory only when they do not fit on chip
    FrameCol frames;
    if(FS)
        frames.p = smem + off * BS + tid, off += 7 * P.L;
    else
        frames.p = lf;

    const double* seed = S.seeds + (size_t)q * P.n_vars;
    const bool do_memetic = active && (phases & PH_MEMETIC) && S.memetic;
    const bool unrolled = has_unrolled_memetic(P);
    // individual 1 and the two gradient vectors only pass through the species block; they can be fetched up front
    // unless the general memetic loop below needs temp / grad as scratch
    const bool species_prefetch = active && (phases & PH_SPECIES) && (!do_memetic || unrolled);
    if(active)
    {
        const double* g = S.goal_params + (size_t)q * G * GOAL_NPARAM;
        for(int k = 0; k < G * GOAL_NPARAM; k++) stage8(&gp[k], g + k);
        const double* gi = S.genes + ((size_t)task * 2 + 0) * n;
        for(int i = 0; i < n; i++) stage8(&ind[i], gi + i);
        for(int v = 0; v < P.n_vars; v++) stage8(&vars[v], seed + v); // non-gene variables stay at the seed (genesToJointVariables)
        if(do_memetic)
        {
            const double* t0 = S.tip0 + (size_t)task * T * 7;
            for(int k = 0; k < 7 * T; k++) stage8(&tip0[k], t0 + k);
            const double* b0 = S.base + (size_t)task * n;
            for(int i = 0; i < n; i++) stage8(&base[i], b0 + i);
            if(DS)
            {
                const double* d0 = S.delta + (size_t)task * T * n * 7;
                for(int k = 0; k < 7 * T * n; k++) stage8(&delta[k], d0 + k);
            }
        }
        if(species_prefetch)
        {
            const double* g1 = S.genes + ((size_t)task * 2 + 1) * n;
            const double* r0 = S.grads + ((size_t)task * 2 + 0) * n;
            const double* r1 = S.grads + ((size_t)task * 2 + 1) * n;
            for(int i = 0; i < n; i++) stage8(&temp[i], g1 + i), stage8(&grad[i], r0 + i), stage8(&stash[i], r1 + i);
        }
        stage_wait();
    }
    const CSC cgp = gp;

    // ---- MEMETIC (src/ik_evolution_2.cpp:436-570) ----------------------------------------------------
    // One evaluation site: the n+4 evaluations of an iteration run through the same loop body
    //   e = 0        x = genes                    full approximation -> ph2   f2p, fa        (:460-464)
    //   e = 1..n     x = genes + dp e_(e-1)       one-variable update of ph2 -> ph3   gradient[e-1] (:465-474)
    //   e = n+1      x = genes - gradient         full -> ph3                 f1             (:485-488)
    //   e = n+2      x = genes + gradient         full -> ph3                 f3             (:492-495)
    //   e = n+3      x = clip(genes +- gradient * step)  full -> ph2          f4p (primary)  (:525-527 / :554-556)
    if(do_memetic)
    {
        double dp = 0.0000001;                                                                                // :450
        if(S.uniform[(6165936u + (uint32_t)stream_step(S, q, step) * 3u + (uint32_t)slot) & ((1u << 23) - 1)] < 0.5) dp = -dp; // :451 fast_random()
        const bool quad = S.memetic == 'q';
        // Fast path for the plugin's default problem (exactly one primary PoseGoal, one tip): tip frames and goal
        // parameters stay in registers; the Pose goal does not read the genes, so the n one-variable evaluations
        // reduce to 7 FMAs + the goal.  Same operations in the same order as the general loop below.
        const bool single_pose = (G == 1 && T == 1 && P.goals[0].type == G_POSE && !P.goals[0].secondary);
        const bool all_move_tip = unrolled;
        if(all_move_tip && n == 7)
            memetic_single_pose<7>(P, S, ind, delta, CSC(tip0), CSC(base), CSC(gp), dp, quad);
        else if(all_move_tip && n == 6)
            memetic_single_pose<6>(P, S, ind, delta, CSC(tip0), CSC(base), CSC(gp), dp, quad);
        else if(single_pose)
        {
            double pg[8], t0r[7];
#pragma unroll
            for(int k = 0; k < 8; k++) pg[k] = gp[k];
#pragma unroll
            for(int k = 0; k < 7; k++) t0r[k] = tip0[k];
            const double wsq = P.goals[0].weight_sq;
            auto full_frames = [&](double (&F)[7]) {
#pragma unroll
                for(int k = 0; k < 7; k++) F[k] = t0r[k];
                for(int i = 0; i < n; i++)
                {
                    if(!(P.genes[i].tipmask & 1)) continue;
                    const double d = temp[i] - base[i]; // :1086
                    const DeltaCol D = delta + 7 * i;
#pragma unroll
                    for(int k = 0; k < 7; k++) F[k] = BIOIK_FMA(d, D[k], F[k]);
                }
            };
            auto pose = [&](const double (&F)[7]) { return 0.0 + link_goal_value(G_POSE, pg, F) * wsq; }; // sum = 0.0; sum += e * weight_sq
            for(int generation = 0; generation < S.memetic_iters; generation++)
            {
                double F2[7], F3[7];
                for(int i = 0; i < n; i++) temp[i] = ind[i]; // :460
                full_frames(F2);                               // :462
                const double f2p = pose(F2);                   // :463
                const double fa = f2p + 0.0;                   // :464 (no secondary goals)
                for(int i = 0; i < n; i++)                     // :465-474
                {
                    const DeltaCol D = delta + 7 * i;
#pragma unroll
                    for(int k = 0; k < 7; k++) F3[k] = BIOIK_FMA(dp, D[k], F2[k]); // :469
                    double fb = 0.0;
                    fb += pose(F3);
                    fb += 0.0;
                    grad[i] = fb - fa;
                }
                double sum = dp * dp; // :477-482
                for(int i = 0; i < n; i++) sum += BIOIK_FABS(grad[i]);
                const double f = 1.0 / sum * dp;
                for(int i = 0; i < n; i++) grad[i] *= f;
                for(int i = 0; i < n; i++) temp[i] = ind[i] - grad[i]; // :485-488
                full_frames(F3);
                double f1 = 0.0;
                f1 += pose(F3);
                f1 += 0.0;
                const double f2 = fa;
                for(int i = 0; i < n; i++) temp[i] = ind[i] + grad[i]; // :492-495
                full_frames(F3);
                double f3 = 0.0;
                f3 += pose(F3);
                f3 += 0.0;
                if(quad) // :502-506,:525
                {
                    double v1 = (f2 - f1);
                    double v2 = (f3 - f2);
                    double v = (v1 + v2) * 0.5;
                    double a = (v1 - v2);
                    double step_size = v / a;
                    for(int i = 0; i < n; i++) temp[i] = clampd(ind[i] + grad[i] * step_size * 1.0, P.genes[i].clip_min, P.genes[i].clip_max);
                }
                else // :549-554
                {
                    double cost_diff = (f3 - f1) * 0.5;
                    double step_size = f2 / cost_diff;
                    for(int i = 0; i < n; i++) temp[i] = clampd(ind[i] - grad[i] * step_size, P.genes[i].clip_min, P.genes[i].clip_max);
                }
                full_frames(F2); // :526 / :555
                const double f4p = pose(F2);
                if(f4p < f2p) // :530-538 / :559-567
                {
                    for(int i = 0; i < n; i++) ind[i] = temp[i];
                    continue;
                }
                else
                    break;
            }
        }
        else
        for(int generation = 0; generation < S.memetic_iters; generation++)
        {
            double f2p = 0.0, fa = 0.0, f1 = 0.0, f3 = 0.0, f4p = 0.0;
            for(int i = 0; i < n; i++) temp[i] = ind[i]; // :460
            for(int e = 0; e < n + 4; e++)
            {
                const bool single = (e >= 1 && e <= n);
                if(single)
                    temp[e - 1] = ind[e - 1] + dp; // :468
                else if(e == n + 1)
                {
                    // normalise the gradient (:477-482), then the first support point (:485-486)
                    double sum = dp * dp;
                    for(int i = 0; i < n; i++) sum += BIOIK_FABS(grad[i]);
                    double f = 1.0 / sum * dp;
                    for(int i = 0; i < n; i++) grad[i] *= f;
                    for(int i = 0; i < n; i++) temp[i] = ind[i] - grad[i];
                }
                else if(e == n + 2)
                    for(int i = 0; i < n; i++) temp[i] = ind[i] + grad[i]; // :492-493
                else if(e == n + 3)
                {
                    const double f2 = fa;
                    if(quad) // :502-506,:525
                    {
                        double v1 = (f2 - f1);
                        double v2 = (f3 - f2);
                        double v = (v1 + v2) * 0.5;
                        double a = (v1 - v2);
                        double step_size = v / a;
                        for(int i = 0; i < n; i++) temp[i] = clampd(ind[i] + grad[i] * step_size * 1.0, P.genes[i].clip_min, P.genes[i].clip_max);
                    }
                    else // :549-554
                    {
                        double cost_diff = (f3 - f1) * 0.5;
                        double step_size = f2 / cost_diff;
                        for(int i = 0; i < n; i++) temp[i] = clampd(ind[i] - grad[i] * step_size, P.genes[i].clip_min, P.genes[i].clip_max);
                    }
                }
                // genotype -> phenotype
                const bool to_ph2 = (e == 0 || e == n + 3);
                const SC out = to_ph2 ? ph2 : ph3;
                if(single)
                    approx_frames1(T, n, delta, e - 1, dp, CSC(ph2), ph3); // :469
                else
                    approx_frames_sparse(P, CSC(tip0), delta, CSC(base), CSC(temp), out); // :462,:487,:494,:526
                // fitness: primary + secondary (computeCombinedFitnessActiveVariables, src/ik_base.h:179-185)
                const double prim = goal_fitness_t(P, 0, cgp, CSC(out), CSC(temp), seed);
                double comb = prim;
                if(e != n + 3) comb = prim + (P.has_secondary ? goal_fitness_secondary(P, cgp, CSC(temp), seed) : 0.0);
                if(e == 0)
                {
                    f2p = prim;
                    fa = comb;
                }
                else if(single)
                {
                    temp[e - 1] = ind[e - 1]; // :471
                    grad[e - 1] = comb - fa;  // :472-473
                }
                else if(e == n + 1)
                    f1 = comb;
                else if(e == n + 2)
                    f3 = comb;
                else
                    f4p = prim;
            }
            if(f4p < f2p) // :530-538 / :559-567
            {
                for(int i = 0; i < n; i++) ind[i] = temp[i];
                continue;
            }
            else
                break;
        }
    }

    // ---- SPECIES (src/ik_evolution_2.cpp:604-645) --------------------------------------------------------
    int my_task = task;        // where this thread's species lives after the sort
    bool frames_valid = false; // `frames` holds the exact FK of `ind`
    if(phases & PH_SPECIES)
    {
        double f = 0.0;
        if(active)
        {
            assemble_genes(P, CSC(ind), vars); // genesToJointVariables :610
            exact_fk(P, CSC(vars), frames);     // computeFitness :611 -> applyConfiguration
            copy_tips(P, frames, ph2);
            f = goal_fitness_t(P, 0, cgp, CSC(ph2), CSC(ind), seed);
            frames_valid = true;
        }
        const double fo = __shfl_xor_sync(0xffffffffu, f, 1);
        int improved = 0, nslot = slot;
        if(active)
        {
            improved = (f != S.sfit[task]) ? 1 : 0; // :612
            // :617 sort ascending: the two species swap places iff species[1].fitness < species[0].fitness
            const bool swap = slot == 0 ? (fo < f) : (f < fo);
            nslot = swap ? (slot ^ 1) : slot;
            my_task = 2 * q + nslot;
            // the rest of this species (individual 1, both gradient vectors) before anybody overwrites it
            const double* g1 = S.genes + ((size_t)task * 2 + 1) * n;
            const double* r0 = S.grads + ((size_t)task * 2 + 0) * n;
            const double* r1 = S.grads + ((size_t)task * 2 + 1) * n;
            if(!species_prefetch)
                for(int i = 0; i < n; i++)
                {
                    temp[i] = g1[i];
                    grad[i] = r0[i];
                    stash[i] = r1[i];
                }
        }
        __syncwarp(); // both species of a query have read their state
        if(active)
        {
            S.sfit[my_task] = f;
            S.impr[my_task] = improved;
            if(nslot == 1)
            {
                // :620-637 wipeout of species[1]; then the random_index draws of the next step's generations (:369)
                uint32_t rng = S.rng[q];
                const double u = S.uniform[(6165936u + (uint32_t)stream_step(S, q, step) * (S.memetic ? 3u : 1u) + (S.memetic ? 2u : 0u)) & ((1u << 23) - 1)];
                if(u < 0.1 || !improved)
                {
                    for(int i = 0; i < n; i++)
                    {
                        double g = minstd_random(rng, P.genes[i].vmin, P.genes[i].vmax); // :629
                        ind[i] = g;
                        temp[i] = g; // individuals[i] = individuals[0]
                        grad[i] = 0.0;
                        stash[i] = 0.0;
                    }
                    frames_valid = false;
                }
                if(P.has_secondary)
                    for(int sl = 0; sl < 2; sl++)
                        for(int g = 0; g < S.gens; g++) S.ccount[((size_t)q * 2 + sl) * S.gens + g] = (int32_t)minstd_index(rng, (uint32_t)(S.C - 3)) + 3;
                S.rng[q] = rng;
            }
            else
            {
                // :640-644 solution update, then the driver's test (src/ik_parallel.h:165-181)
                bool sol_is_ind = false;
                if(f < S.solfit[q])
                {
                    for(int i = 0; i < n; i++) S.sol[(size_t)q * n + i] = ind[i];
                    S.solfit[q] = f;
                    sol_is_ind = true;
                }
                const int steps = S.steps[q] + 1;
                S.steps[q] = steps;
                if((steps % 4) == 0 || steps == S.total_steps)
                {
                    // getSolution() -> exact FK -> checkSolution.  If the solution is this species' individual
                    // its exact tip frames are already in ph2; otherwise recompute them (frames/vars are scratch).
                    // grads of individual 1 are parked in `stash`, individual 1 genes in `temp`: use base/ph3.
                    SC xs = ind, ts = ph2;
                    if(!sol_is_ind)
                    {
                        const double* sol = S.sol + (size_t)q * n;
                        for(int i = 0; i < n; i++) base[i] = sol[i];
                        assemble_genes(P, CSC(base), vars);
                        exact_fk(P, CSC(vars), frames);
                        copy_tips(P, frames, ph3);
                        frames_valid = false;
                        xs = base;
                        ts = ph3;
                    }
                    const int ok = check_solution(P, cgp, CSC(ts), CSC(xs), seed) ? 1 : 0;
                    S.success[q] = ok;
                    if(ok) note_success(S, q, steps);
                }
            }
            // write the species back (to its new slot)
            double* og0 = S.genes + ((size_t)my_task * 2 + 0) * n;
            double* og1 = S.genes + ((size_t)my_task * 2 + 1) * n;
            double* or0 = S.grads + ((size_t)my_task * 2 + 0) * n;
            double* or1 = S.grads + ((size_t)my_task * 2 + 1) * n;
            for(int i = 0; i < n; i++)
            {
                og0[i] = ind[i];
                og1[i] = temp[i];
                or0[i] = grad[i];
                or1[i] = stash[i];
            }
        }
    }
    else if(active && (phases & PH_MEMETIC))
    {
        double* og0 = S.genes + ((size_t)task * 2 + 0) * n;
        for(int i = 0; i < n; i++) og0[i] = ind[i];
    }

    // ---- PREPARE (src/ik_evolution_2.cpp:341-346) ---------------------------------------------------------
    if(active && (phases & PH_PREPARE))
    {
        // p_variables = post-mimic variables of the base configuration (:1063)
        assemble_genes(P, CSC(ind), vars);
        if(!frames_valid) exact_fk(P, CSC(vars), frames);
        double* t0 = S.tip0 + (size_t)my_task * T * 7;
        for(int t = 0; t < T; t++)
            for(int k = 0; k < 7; k++) t0[7 * t + k] = frames[7 * P.tip_slot[t] + k];
        double* b0 = S.base + (size_t)my_task * n;
        for(int i = 0; i < n; i++) b0[i] = vars[P.genes[i].var];
        double* d0 = S.delta + (size_t)my_task * T * n * 7;
        for(int t = 0; t < T; t++)
            for(int i = 0; i < n; i++)
            {
                F7 df;
                if((P.genes[i].tipmask >> t) & 1)
                {
                    bool masked;
                    df = delta_frame(P, frames, CSC(vars), i, t, masked);
                }
                else // structurally independent pair: the Jacobian column is exactly zero (:609-617), so is the delta frame
                    df = F7{{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0, 0.0}};
                store_frame(d0 + ((size_t)t * n + i) * 7, df);
            }
    }
}

template <int BS, bool DS, bool FS> __global__ void __launch_bounds__(BS) k_serial(BIOIK_PROBLEM_PARAM, DState S, int step, int phases)
{
    extern __shared__ double smem[];
    serial_tasks<BS, DS, FS>(P, S, step, phases, smem, threadIdx.x, blockIdx.x * BS + threadIdx.x);
}

#ifdef BIOIK_HOSTSIM
typedef void (*SerialKernel)(const DProblem&, DState, int, int);
#else
typedef void (*SerialKernel)(const DProblem, DState, int, int);
#endif

inline SerialKernel select_serial(const SerialPlan& pl)
{
#ifdef BIOIK_SLIM // experiment builds: the headline shape only (fast compile)
    return (SerialKernel)k_serial<32, true, false>;
#else
#define BIOIK_SER(BS)                                                                                                            \
    (pl.delta_smem ? (pl.frames_smem ? (SerialKernel)k_serial<BS, true, true> : (SerialKernel)k_serial<BS, true, false>) \
                   : (pl.frames_smem ? (SerialKernel)k_serial<BS, false, true> : (SerialKernel)k_serial<BS, false, false>))
    switch(pl.block)
    {
    case 128: return BIOIK_SER(128);
    case 64: return BIOIK_SER(64);
    default: return BIOIK_SER(32);
    }
#undef BIOIK_SER
#endif
}

} // namespace bioik
