// bioik_memetic_group.cuh — the memetic line search (src/ik_evolution_2.cpp:436-570) with a GROUP of W lanes
// per task instead of one thread (DESIGN.md §6).
//
// An iteration of the reference is n+4 dependent-looking evaluations, but only four of them depend on each
// other:   f2p  ->  { n gradient probes }  ->  { f1, f3 }  ->  f4p
// and a full approximation (computeApproximateMutations, forward_kinematics.h:1061-1110) is 7T independent
// FMA chains.  The group therefore runs
//   * the 7T (or 2 x 7T) frame components of a full approximation on 7T (14T) lanes,
//   * the n one-variable probes (computeApproximateMutation1 + combined fitness) on n lanes,
//   * the element-wise gene / gradient updates on n lanes,
// while every VALUE is produced by the same operations in the same order as in the thread-per-task kernel
// (k_serial, PH_MEMETIC) — the two are interchangeable bit for bit (tests/test_hostsim_parity.py).
// The thread-per-task version left the SMs with one warp or less each (B = 10 000 queries -> 625 warps on 132 SMs)
// and paid the full latency of every FP64 operation; here the same batch is 5 000 warps at W = 8.
#pragma once

#include "bioik_dev.cuh"
#include "bioik_serial.cuh"

namespace bioik
{

// The joint-space goals that are a sum over the active variables (goal_types.h:387-465): sum = 0, then sum += term(gene)
// for every gene the goal applies to, in gene order.  term() is the loop body of goal_value's case, operation for operation.
BIOIK_HD bool is_summing_joint_goal(int type) { return type == G_AVOID_JOINT_LIMITS || type == G_CENTER_JOINTS || type == G_REGULARIZATION || type == G_MINIMAL_DISPLACEMENT; }
BIOIK_HD bool joint_term_applies(const DProblem& P, int type, int i) { return (type == G_AVOID_JOINT_LIMITS || type == G_CENTER_JOINTS) ? P.genes[i].clip_max != DBLMAX : true; }
// term() per goal type (x = the variable's value), with r = {centre, half span, weight, avoid} built once per task:
//   AvoidJointLimitsGoal  d = x - (min + max) / 2;  d = max(0, |d| * 2 - span / 2);  d *= weight     goal_types.h:387-401
//   CenterJointsGoal      d = x - (min + max) / 2;  d *= weight                                        goal_types.h:412-425
//   RegularizationGoal    d = x - seed                                                                 goal_types.h:435-444
//   MinimalDisplacement   d = x - seed;  d *= weight                                                   goal_types.h:455-465
// and the term is d * d.  A lane asks for the term of ITS variable, so reading DProblem::genes[i] / seed[var] at that point would
// be a lane-divergent constant-bank access plus a global load per call (the top stall of this kernel on cfg4 before the records).
// RegularizationGoal has no weight factor: * 1.0 is exact.
BIOIK_HD double joint_term_rec(const double* r, double x)
{
    double d = x - r[0];
    if(r[3] != 0.0) d = BIOIK_FMAX(0.0, BIOIK_FABS(d) * 2.0 - r[1]);
    d *= r[2];
    return d * d;
}

// genes of a probe: individual.genes with element i replaced (ik_evolution_2.cpp:468-471)
struct ProbeGenes
{
    const double* ind;
    int i;
    double v;
    BIOIK_HD double operator[](int k) const { return k == i ? v : ind[k]; }
};

// the one tip frame a link goal of a probe reads, held in registers (goal_value offsets its frame argument by 7 * tip)
struct ProbeFrame
{
    const double* f;
    BIOIK_HD ProbeFrame operator+(int) const { return *this; }
    BIOIK_HD double operator[](int k) const { return f[k]; }
};

// shared-memory block of one group, in doubles.  K = number of (tip, gene) pairs where the gene can move the tip
// (DProblem::tip_gene; every other delta frame is all zero and never read)
struct GroupLayout
{
    int n, T, G, W, K, stale, NJ; // NJ = joint-space goals of the problem (an upper bound of the summing ones)
    __host__ __device__ int o_ind() const { return 0; }
    __host__ __device__ int o_graw() const { return n; }
    __host__ __device__ int o_grad() const { return 2 * n; }
    __host__ __device__ int o_ta() const { return 3 * n; }
    __host__ __device__ int o_tb() const { return 4 * n; }
    __host__ __device__ int o_base() const { return 5 * n; }
    __host__ __device__ int o_clip() const { return 6 * n; } // [n][2]
    __host__ __device__ int o_tip0() const { return 8 * n; }
    __host__ __device__ int o_f2() const { return o_tip0() + 7 * T; }
    __host__ __device__ int o_pl() const { return o_f2() + 7 * T; }     // [2][7T] frames of the two support points
    __host__ __device__ int o_delta() const { return o_pl() + 14 * T; } // [K][7] delta frames in pair order (tip-major, genes ascending)
    __host__ __device__ int o_dxa() const { return o_delta() + 7 * K; } // [K] x - base of the pair's gene: current genes / support point a / candidate
    __host__ __device__ int o_dxb() const { return o_dxa() + K; }       // [K] the same for support point b
    __host__ __device__ int o_gp() const { return o_dxb() + K; }
    __host__ __device__ int o_gv() const { return o_gp() + GOAL_NPARAM * G; } // [3][G] goal values: current genes; support point a / candidate; support point b
    __host__ __device__ int o_sc() const { return o_gv() + 3 * G; }
    __host__ __device__ int o_carry() const { return o_sc() + 8; }               // [7T] reference-quirk mode: the frames left in phenotypes3
    __host__ __device__ int o_jt() const { return o_carry() + (stale ? 7 * T : 0); } // [3][NJ][n] terms of the summing joint-space goals, rows as gv
    __host__ __device__ int o_jr() const { return o_jt() + 3 * NJ * n; }             // [NJ][n][4] records of joint_term_rec (rows as jt's slots)
    __host__ __device__ int o_int() const { return o_jr() + 4 * NJ * n; }
    // int32: pair_start [T + 1], pair_gene [K], pair_of [T][n] (-1: the gene cannot move the tip), sum_slot [G] (row of jt, -1: not a
    // summing joint-space goal); reference-quirk mode: prev_pair [T][n] = pair of the last earlier gene that moves tip t (-1: none)
    __host__ __device__ int ints() const { return T + 1 + K + T * n + G + (stale ? T * n : 0); }
    __host__ __device__ int total() const { return (o_int() + (ints() + 1) / 2) | 1; } // odd stride: the groups of a warp start in different banks
};

inline int memetic_group_width(int n) { return n <= 8 ? 8 : (n <= 16 ? 16 : 32); }

// W lanes per task, 32 / W tasks per warp; blockDim.x = 32 * warps (any number of warps, no block-level sync)
//
// Schedule of one iteration (values as in the thread-per-task kernel, see the header):
//   * a full approximation = 7T FMA chains, each over the pairs of its tip only, on 7T lanes; x - base (:1086) is formed once
//     per pair by the phase that produces x;
//   * Goal::evaluate of every goal on its own lane, then the weighted sum in goal order on one lane (src/problem.cpp:251-257);
//   * a probe builds the one frame each link goal reads in registers (computeApproximateMutation1 of ONE variable);
//   * a joint-space goal that sums over the variables has its terms formed by the lane of each variable where the variable's
//     value is produced; the evaluation is the ordered sum of the stored terms (a probe substitutes its one term);
//   * the candidate of an accepted iteration IS the next iteration's individual: its frames and goal values (f4p, and the
//     secondary goals for fa) are kept instead of being recomputed by (1) and (2).
//
// STALE = the reference-quirk mode (bioik_set_option BIOIK_OPT_REFERENCE_STALE_TIPS, SURVEY.md Q2): the reference's
// computeApproximateMutation1 skips the tips a variable cannot move (forward_kinematics.h:940), so a probe scores those
// tips on what phenotypes3[0] held before: the frame written by the last earlier probe of the iteration that moves the tip,
// else the frames of the previous f3 evaluation (:494) - of the previous iteration, of the other species (the solver has ONE
// phenotypes3 and treats species 0, then species 1), or of the previous step.  Here a group owns a QUERY, runs its two
// species one after the other and carries those frames in `carry` (HBM between steps; identity frames at the start, which
// is what the harness of the reference build pre-fills - a fresh reference solver reads uninitialised memory there).
// blocks per SM the register allocation aims for: the kernel is a chain of short dependent phases (latency-bound), so more
// resident warps beat a larger register file per thread (80 registers, no spills)
// (the 16-lane form - two tasks per warp, problems of 9 ... 16 variables - is the exception: four blocks with 128 registers run cfg3's
// memetic phase faster than six; the 32-lane form loses that way)
#ifndef BIOIK_MG_MINBLOCKS
#define BIOIK_MG_MINBLOCKS 6
#endif
template <int W, bool STALE = false> __global__ void __launch_bounds__(128, (W == 16 ? 4 : BIOIK_MG_MINBLOCKS)) k_memetic_group(BIOIK_PROBLEM_PARAM, DState S, int step)
{
    extern __shared__ double smem[];
    constexpr int GPW = 32 / W;
    constexpr unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31, warp_in_block = threadIdx.x >> 5, warps_per_block = blockDim.x >> 5;
    const int gl = lane % W, gw = lane / W;
    const int unit_raw = (blockIdx.x * warps_per_block + warp_in_block) * GPW + gw; // task (query, slot), or query in STALE mode
    const int units = STALE ? S.B : 2 * S.B;
    const bool valid = unit_raw < units;
    const int unit = valid ? unit_raw : units - 1;
    const int q = STALE ? unit : (unit >> 1);
    const bool live = valid && !run_done(S, q, step) && S.memetic;
    const int n = P.n, T = P.T, G = P.G, T7 = 7 * P.T, K = P.tip_gene_start[P.T];

    const GroupLayout L{n, T, G, W, K, STALE ? 1 : 0, P.n_joint_goals};
    const int NJ = P.n_joint_goals;
    double* Wk = smem + (size_t)(warp_in_block * GPW + gw) * L.total();
    double *ind = Wk + L.o_ind(), *graw = Wk + L.o_graw(), *grad = Wk + L.o_grad(), *ta = Wk + L.o_ta(), *tb = Wk + L.o_tb(), *base = Wk + L.o_base(), *clip = Wk + L.o_clip();
    double *tip0 = Wk + L.o_tip0(), *f2 = Wk + L.o_f2(), *pl = Wk + L.o_pl(), *delta = Wk + L.o_delta(), *dxa = Wk + L.o_dxa(), *dxb = Wk + L.o_dxb();
    double *gp = Wk + L.o_gp(), *gv = Wk + L.o_gv(), *sc = Wk + L.o_sc(), *carry = Wk + L.o_carry(), *jt = Wk + L.o_jt(), *jr = Wk + L.o_jr();
    int32_t* pair_start = (int32_t*)(Wk + L.o_int());
    int32_t *pair_gene = pair_start + T + 1, *pair_of = pair_gene + K, *sum_slot = pair_of + T * n, *prev_pair = sum_slot + G;
    const double* seed = S.seeds + (size_t)q * P.n_vars;
    // terms of the summing joint-space goals for gene i at value x -> row of jt
    auto store_terms = [&](int row, int i, double x) {
        for(int g = 0; g < G; g++)
            if(sum_slot[g] >= 0) jt[((size_t)row * NJ + sum_slot[g]) * n + i] = joint_term_rec(jr + ((size_t)sum_slot[g] * n + i) * 4, x);
    };

    // the pair lists of the problem, next to the data they index
    if(live)
    {
        for(int t = gl; t <= T; t += W) pair_start[t] = P.tip_gene_start[t];
        for(int k = gl; k < K; k += W) pair_gene[k] = P.tip_gene[k];
        for(int k = gl; k < T * n; k += W) pair_of[k] = -1;
        for(int g = gl; g < G; g += W)
        {
            int slot = 0;
            for(int h = 0; h < g; h++) slot += is_summing_joint_goal(P.goals[h].type) ? 1 : 0;
            sum_slot[g] = is_summing_joint_goal(P.goals[g].type) ? slot : -1;
        }
    }
    __syncwarp();
    if(live)
    {
        for(int k = gl; k < K; k += W)
        {
            int t = 0;
            while(pair_start[t + 1] <= k) t++;
            pair_of[t * n + pair_gene[k]] = k;
        }
        for(int g = 0; g < G; g++)
        {
            if(sum_slot[g] < 0) continue;
            const int type = P.goals[g].type;
            for(int i = gl; i < n; i += W)
            {
                const DGene& Gn = P.genes[i];
                const bool limits = type == G_AVOID_JOINT_LIMITS || type == G_CENTER_JOINTS;
                double* r = jr + ((size_t)sum_slot[g] * n + i) * 4;
                r[0] = limits ? (Gn.vmin + Gn.vmax) * 0.5 : seed[Gn.var];
                r[1] = Gn.span * 0.5;
                r[2] = type == G_REGULARIZATION ? 1.0 : Gn.vel_weight;
                r[3] = type == G_AVOID_JOINT_LIMITS ? 1.0 : 0.0;
            }
        }
    }
    __syncwarp();
    if(STALE && live)
    {
        for(int c = gl; c < T7; c += W) carry[c] = S.carry[(size_t)q * T7 + c];
        for(int k = gl; k < T * n; k += W)
        {
            const int t = k / n, i = k - t * n;
            int j = i - 1;
            while(j >= 0 && pair_of[t * n + j] < 0) j--;
            prev_pair[k] = j >= 0 ? pair_of[t * n + j] : -1;
        }
    }
    for(int slot_it = 0; slot_it < (STALE ? 2 : 1); slot_it++)
    {
    const int task = STALE ? 2 * q + slot_it : unit;
    const int slot = task & 1;
    bool alive = live;

    // ---- stage the task ------------------------------------------------------------------------
    if(alive)
    {
        const double* g = S.goal_params + (size_t)q * G * GOAL_NPARAM;
        for(int k = gl; k < G * GOAL_NPARAM; k += W) gp[k] = g[k];
        const double* gi = S.genes + ((size_t)task * 2 + 0) * n;
        const double* b0 = S.base + (size_t)task * n;
        for(int i = gl; i < n; i += W)
        {
            ind[i] = gi[i];
            base[i] = b0[i];
            clip[2 * i + 0] = P.genes[i].clip_min;
            clip[2 * i + 1] = P.genes[i].clip_max;
        }
        const double* t0 = S.tip0 + (size_t)task * T * 7;
        for(int k = gl; k < T7; k += W) tip0[k] = t0[k];
        const double* d0 = S.delta + (size_t)task * T * n * 7;
        for(int k = gl; k < 7 * K; k += W)
        {
            const int idx = k / 7, c = k - 7 * idx;
            int t = 0;
            while(pair_start[t + 1] <= idx) t++;
            delta[k] = d0[((size_t)t * n + pair_gene[idx]) * 7 + c];
        }
        for(int idx = gl; idx < K; idx += W) dxa[idx] = gi[pair_gene[idx]] - b0[pair_gene[idx]]; // :1086
        if(NJ)
            for(int i = gl; i < n; i += W) store_terms(0, i, gi[i]);
    }
    __syncwarp();

    double dp = 0.0000001;                                                                                // :450
    if(S.uniform[(6165936u + (uint32_t)stream_step(S, q, step) * 3u + (uint32_t)slot) & ((1u << 23) - 1)] < 0.5) dp = -dp; // :451 fast_random()
    const bool quad = S.memetic == 'q';

    // component c (= 7 t + k) of the full approximation of a genotype x given as dx = x - base per pair: the FMA chain of
    // approx_frames_sparse (the pairs of tip t in ascending gene order)
    auto chain = [&](const double* dx, int c) {
        const int t = c / 7;
        double f = tip0[c];
        const double* D = delta + (c - 7 * t);
        const int i1 = pair_start[t + 1];
        for(int idx = pair_start[t]; idx < i1; idx++) f = BIOIK_FMA(dx[idx], D[7 * idx], f);
        return f;
    };
    // Goal::evaluate of goal g for the genes x whose terms are in row `row` of jt; secondary goals see the identity frames
    // (src/ik_base.h:163)
    auto goal_at = [&](int g, const double* frames, const double* x, int row) {
        const DGoal& go = P.goals[g];
        const int slot = sum_slot[g];
        if(slot >= 0)
        {
            const double* t = jt + ((size_t)row * NJ + slot) * n;
            double sum = 0.0;
            for(int i = 0; i < n; i++)
                if(joint_term_applies(P, go.type, i)) sum += t[i];
            return sum;
        }
        return goal_value(P, go, (const double*)gp + g * GOAL_NPARAM, go.secondary ? (const double*)NULL_TIPS : frames, x, seed);
    };
    // the weighted sums of computeFitnessActiveVariables / computeCombinedFitnessActiveVariables (src/ik_base.h:179-185) over a
    // row of goal values, in goal order
    auto goal_sum = [&](int row, int which) {
        double sum = 0.0;
        for(int g = 0; g < G; g++)
            if(P.goals[g].secondary == which) sum += gv[row * G + g] * P.goals[g].weight_sq;
        return sum;
    };

    for(int generation = 0; generation < S.memetic_iters; generation++)
    {
        if(!__any_sync(FULL, alive)) break;
        if(generation == 0)
        {
            // (1) genotype = individual.genes -> phenotypes2 (:460-462)
            if(alive)
                for(int c = gl; c < T7; c += W) f2[c] = chain(dxa, c);
            __syncwarp();
            // (2) f2p, fa (:463-464)
            if(alive)
                for(int g = gl; g < G; g += W) gv[g] = goal_at(g, f2, ind, 0);
            __syncwarp();
            if(alive && gl == 0)
            {
                const double prim = goal_sum(0, 0);
                sc[0] = prim;
                sc[1] = prim + (P.has_secondary ? goal_sum(0, 1) : 0.0);
            }
            __syncwarp();
        }
        // (3) gradient probes (:465-474): lane i moves variable i by dp
        if(alive)
        {
            const double fa = sc[1];
            for(int i = gl; i < n; i += W)
            {
                const ProbeGenes x{ind, i, ind[i] + dp}; // :468
                double prim = 0.0, sec = 0.0;
                for(int g = 0; g < G; g++)
                {
                    const DGoal& go = P.goals[g];
                    double v;
                    if(sum_slot[g] >= 0)
                    {
                        // the stored terms of the current genes with this variable's term replaced
                        const double* t = jt + (size_t)sum_slot[g] * n;
                        const double mine = joint_term_rec(jr + ((size_t)sum_slot[g] * n + i) * 4, x.v);
                        double sum = 0.0;
                        for(int j = 0; j < n; j++)
                            if(joint_term_applies(P, go.type, j)) sum += j == i ? mine : t[j];
                        v = sum;
                    }
                    else if(is_joint_goal(go.type))
                        v = goal_value(P, go, (const double*)gp + g * GOAL_NPARAM, (const double*)NULL_TIPS, x, seed);
                    else if(go.secondary)
                        v = gv[g]; // a link goal on the identity frames: what it is for the current genes
                    else
                    {
                        // :469 for the tip of this goal
                        const int t = go.tip;
                        int pi = pair_of[t * n + i];
                        double fr[7];
                        if(!STALE)
                        {
                            // a tip the variable cannot move stays where the current genes put it (its delta frame is zero)
                            for(int k = 0; k < 7; k++) fr[k] = pi >= 0 ? BIOIK_FMA(dp, delta[7 * pi + k], f2[7 * t + k]) : f2[7 * t + k];
                        }
                        else
                        {
                            // the tip keeps what the buffer held: the write of the last earlier probe that moves it, else the carried frame
                            if(pi < 0) pi = prev_pair[t * n + i];
                            for(int k = 0; k < 7; k++) fr[k] = pi >= 0 ? BIOIK_FMA(dp, delta[7 * pi + k], f2[7 * t + k]) : carry[7 * t + k];
                        }
                        v = goal_value(P, go, (const double*)gp + g * GOAL_NPARAM, ProbeFrame{fr}, x, seed);
                    }
                    if(go.secondary)
                        sec += v * go.weight_sq;
                    else
                        prim += v * go.weight_sq;
                }
                graw[i] = (prim + (P.has_secondary ? sec : 0.0)) - fa; // :472-473
            }
        }
        __syncwarp();
        // (4) normalise (:477-482) and the two support points (:485-486, :492-493)
        if(alive)
        {
            double sum = dp * dp;
            for(int i = 0; i < n; i++) sum += BIOIK_FABS(graw[i]);
            const double f = 1.0 / sum * dp;
            for(int i = gl; i < n; i += W)
            {
                const double g = graw[i] * f;
                grad[i] = g;
                ta[i] = ind[i] - g;
                tb[i] = ind[i] + g;
                if(NJ) store_terms(1, i, ind[i] - g), store_terms(2, i, ind[i] + g);
            }
            for(int idx = gl; idx < K; idx += W)
            {
                const int i = pair_gene[idx];
                const double g = graw[i] * f;
                dxa[idx] = (ind[i] - g) - base[i]; // :1086
                dxb[idx] = (ind[i] + g) - base[i];
            }
        }
        __syncwarp();
        // (5) both support points -> frames
        if(alive)
            for(int c = gl; c < 2 * T7; c += W)
            {
                const int which = c >= T7 ? 1 : 0;
                pl[c] = chain(which ? dxb : dxa, c - which * T7);
            }
        __syncwarp();
        // (6) f1, f3 (:487-488, :494-495)
        if(alive)
            for(int item = gl; item < 2 * G; item += W)
            {
                const int which = item >= G ? 1 : 0;
                gv[G + item] = goal_at(item - which * G, pl + which * T7, which ? tb : ta, 1 + which);
            }
        __syncwarp();
        if(alive && gl < 2) sc[2 + gl] = goal_sum(1 + gl, 0) + (P.has_secondary ? goal_sum(1 + gl, 1) : 0.0);
        __syncwarp();
        // (7) step size and the candidate (:502-506,:525 / :549-554)
        if(alive)
        {
            if(STALE)
                for(int c = gl; c < T7; c += W) carry[c] = pl[T7 + c]; // phenotypes3 now holds the frames of the f3 evaluation (:494)
            const double f2v = sc[1], f1 = sc[2], f3 = sc[3];
            double step_size;
            if(quad)
            {
                double v1 = (f2v - f1);
                double v2 = (f3 - f2v);
                double v = (v1 + v2) * 0.5;
                double a = (v1 - v2);
                step_size = v / a;
                for(int i = gl; i < n; i += W)
                {
                    ta[i] = clampd(ind[i] + grad[i] * step_size * 1.0, clip[2 * i], clip[2 * i + 1]);
                    if(NJ) store_terms(1, i, ta[i]);
                }
                for(int idx = gl; idx < K; idx += W)
                {
                    const int i = pair_gene[idx];
                    dxa[idx] = clampd(ind[i] + grad[i] * step_size * 1.0, clip[2 * i], clip[2 * i + 1]) - base[i];
                }
            }
            else
            {
                double cost_diff = (f3 - f1) * 0.5;
                step_size = f2v / cost_diff;
                for(int i = gl; i < n; i += W)
                {
                    ta[i] = clampd(ind[i] - grad[i] * step_size, clip[2 * i], clip[2 * i + 1]);
                    if(NJ) store_terms(1, i, ta[i]);
                }
                for(int idx = gl; idx < K; idx += W)
                {
                    const int i = pair_gene[idx];
                    dxa[idx] = clampd(ind[i] - grad[i] * step_size, clip[2 * i], clip[2 * i + 1]) - base[i];
                }
            }
        }
        __syncwarp();
        // (8) candidate -> phenotypes2 (:526 / :555)
        if(alive)
            for(int c = gl; c < T7; c += W) f2[c] = chain(dxa, c);
        __syncwarp();
        // (9) f4p - and the candidate's secondary goals: if it is accepted they are the next iteration's fa
        if(alive)
            for(int g = gl; g < G; g += W) gv[G + g] = goal_at(g, f2, ta, 1);
        __syncwarp();
        if(alive && gl == 0) sc[4] = goal_sum(1, 0);
        __syncwarp();
        // (10) accept / stop (:530-538 / :559-567)
        bool accept = false;
        if(alive) accept = sc[4] < sc[0];
        __syncwarp();
        if(alive)
        {
            if(accept)
            {
                // individual.genes = candidate: phenotypes2, f2p and fa of the next iteration (:460-464) are the candidate's
                for(int i = gl; i < n; i += W) ind[i] = ta[i];
                for(int k = gl; k < NJ * n; k += W) jt[k] = jt[NJ * n + k];
                for(int g = gl; g < G; g += W) gv[g] = gv[G + g];
                if(gl == 0)
                {
                    sc[0] = sc[4];
                    sc[1] = sc[4] + (P.has_secondary ? goal_sum(1, 1) : 0.0);
                }
            }
            else
                alive = false;
        }
        __syncwarp();
    }

    // individuals[0].genes back to the state (gradients are not touched by the memetic step)
    if(live)
    {
        double* og0 = S.genes + ((size_t)task * 2 + 0) * n;
        for(int i = gl; i < n; i += W) og0[i] = ind[i];
    }
    __syncwarp(); // the next species of the query re-uses the block
    } // species of the query (STALE), or the single task
    if(STALE && live)
        for(int c = gl; c < T7; c += W) S.carry[(size_t)q * T7 + c] = carry[c];
}

#ifdef BIOIK_HOSTSIM
typedef void (*MemeticGroupKernel)(const DProblem&, DState, int);
#else
typedef void (*MemeticGroupKernel)(const DProblem, DState, int);
#endif

inline MemeticGroupKernel select_memetic_group(int W, bool stale = false)
{
#ifdef BIOIK_SLIM
    return (MemeticGroupKernel)k_memetic_group<8>;
#else
    if(stale) return W == 8 ? (MemeticGroupKernel)k_memetic_group<8, true> : (W == 16 ? (MemeticGroupKernel)k_memetic_group<16, true> : (MemeticGroupKernel)k_memetic_group<32, true>);
    return W == 8 ? (MemeticGroupKernel)k_memetic_group<8> : (W == 16 ? (MemeticGroupKernel)k_memetic_group<16> : (MemeticGroupKernel)k_memetic_group<32>);
#endif
}

// the reference-quirk mode changes something only if some gene cannot move some tip
__host__ __device__ inline bool stale_tips_matter(const DProblem& P)
{
    for(int i = 0; i < P.n; i++)
        if((P.genes[i].tipmask & ((1 << P.T) - 1)) != ((1 << P.T) - 1)) return true;
    return false;
}

} // namespace bioik
