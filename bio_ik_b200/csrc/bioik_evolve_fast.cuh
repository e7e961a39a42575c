// bioik_evolve_fast.cuh — register-blocked generation kernel (the dominant kernel).
//
// Same arithmetic as k_evolve / the reference (src/ik_evolution_2.cpp:351-432), different
// schedule (DESIGN.md §5):
//   * one warp per task, lane l owns child slots l, l+32, ... (CPL of them) and evaluates
//     them TOGETHER: per gene the warp-uniform operands (parent gene, limits, base, delta
//     frame) are read once from shared memory and applied to CPL children, tip-frame
//     accumulators live in registers, genes are never stored;
//   * the mutation term r * (mutation_rate * span) of every (reproduce call, gene, child)
//     is query-independent — gaussians and rate exponents are consumed in a fixed order
//     (src/ik_evolution_2.cpp:254-265,288-293) — so it is tabulated once per problem
//     (k_mutation_table) in a [call][gene][child] layout: lanes read consecutive doubles;
//   * joint-space goals (sums over genes) are accumulated inside the gene loop in gene
//     order, link goals are evaluated from the register tip frames; goal order of the
//     final weighted sum is kept (src/problem.cpp:251-257);
//   * the two winners are re-derived from the table instead of storing 2*n doubles per child.
#pragma once

#include "bioik_dev.cuh"

#include <type_traits>

#ifdef BIOIK_HOSTSIM
#define BIOIK_LDG(p) (*(p))
#else
#define BIOIK_LDG(p) __ldg(p)
#endif

// 1: the single-pose kernels request the first mutation-table row of a chunk one chunk ahead (evolve_fast_task, EARLY)
#ifndef BIOIK_EVOLVE_EARLYROW
#define BIOIK_EVOLVE_EARLYROW 0
#endif

namespace bioik
{

constexpr int FAST_MAX_JOINT_GOALS = 4;

// row length of the mutation table: child slots 2..C-1 re-indexed j = c - 2 and padded to whole warps
// to a power of two >= 32 (32, 64, 128 or 256) so that every register-block size divides it
__host__ __device__ inline int mtab_row(int C)
{
    int r = 32;
    while(r < C - 2) r *= 2;
    return r;
}

// mutation table: mtab[(call * n + gene) * mtab_row(C) + j] = r * (mutation_rate * span), j = child - 2   (:288-293)
// (zero in the padding, so padded lanes read valid memory and their results are simply never selected)
__global__ void k_mutation_table(const DProblem* __restrict__ Pp, int calls, int C, const double* __restrict__ gauss, const int32_t* __restrict__ gauss_off, const uint8_t* __restrict__ rate_exp, double* __restrict__ mtab)
{
    const DProblem& P = *Pp;
    const int n = P.n, R = mtab_row(C);
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long total = (long long)calls * n * R;
    if(idx >= total) return;
    int j = (int)(idx % R);
    int i = (int)((idx / R) % n);
    int call = (int)(idx / ((long long)R * n));
    double m = 0.0;
    if(j < C - 2)
    {
        const int stride4 = (n + 3) / 4 * 4;
        double r = gauss[gauss_off[call] + (size_t)j * stride4 + i];
        double mutation_rate = (double)(1 << rate_exp[(size_t)call * (C - 2) + j]) * (1.0 / (double)(1 << 23)); // :265
        double f = mutation_rate * P.genes[i].span;                                                            // :290
        m = r * f;                                                                                             // :293
    }
    mtab[idx] = m;
}

// per-warp shared-memory carve-up (doubles); every block is 16-byte aligned
struct FastSmem
{
    int n, T, G, nj; // nj = joint-space goals of the problem (0: no joint records)
    int lean = 0; // 1: no per-child fitness arrays (only the pre-selection of problems with secondary goals reads them)
    int pairs = 0; // tip-major form: the delta frames of the (tip, gene) pairs of DProblem::tip_gene only, in list order (0: dense [T][n])
    __host__ __device__ int off_rec() const { return 0; }                        // [n][4]  g0, base, clip_min, clip_max
    __host__ __device__ int off_term() const { return off_rec() + 4 * n; }       // [n][6]  pg[parity] * gradient_factor
    __host__ __device__ int off_delta() const { return off_term() + 6 * n; }     // [T][n][8], or [pairs][8]
    __host__ __device__ int off_par() const { return off_delta() + 8 * (pairs ? pairs : T * n); }  // [2 buffers][g0,g1,gr0,gr1][n]
    __host__ __device__ int off_pg() const { return off_par() + 8 * n; }         // [2][n] mix(gr0, gr1, fmix)
    __host__ __device__ int off_tip0() const { return off_pg() + 2 * n; }        // [T][8]
    __host__ __device__ int off_gp() const { return off_tip0() + 8 * T; }        // [G][12]
    __host__ __device__ int off_jrec() const { return off_gp() + 12 * G; }       // [n][4]  mid, halfspan, vel_weight, seed  (nj > 0)
    __host__ __device__ int off_jq() const { return off_jrec() + (nj ? 4 * n : 0); }       // [MAXJ][n][4] joint-goal records: centre, half span, weight, on (nj > 0)
    __host__ __device__ int off_fit() const { return off_jq() + 4 * nj * n; } // [256] primary fitness per child slot
    __host__ __device__ int off_sf() const { return off_fit() + (lean ? 0 : 256); }   // [256] secondary fitness per child slot
    // tip-major form: the warp-uniform operands of the chains in PAIR order, so that the chain loop walks them with pointer bumps
    // instead of indexing by gene: [pairs][4] g0, base, clip_min, clip_max and [pairs][6] the gradient terms (the mutation-table
    // offset gene * row of a pair sits in the pad slot 7 of its delta frame)
    __host__ __device__ int off_prec() const { return off_sf() + (lean ? 0 : 256); }
    __host__ __device__ int off_pterm() const { return off_prec() + 4 * pairs; }
    __host__ __device__ int total() const { return ((off_pterm() + 6 * pairs) + 1) & ~1; }
};

// problems with three or more tips run the tip-major form of the generation kernel (select_evolve_fast)
#ifndef BIOIK_TM_MIN_TIPS
#define BIOIK_TM_MIN_TIPS 3
#endif
__host__ __device__ inline bool fast_tip_major(const DProblem& P) { return P.T >= BIOIK_TM_MIN_TIPS; }
// the shared-memory plan of one task of the generation kernel select_evolve_fast picks for P
__host__ __device__ inline FastSmem fast_smem_layout(const DProblem& P)
{
    return FastSmem{P.n, P.T, P.G, P.n_joint_goals, P.has_secondary ? 0 : 1, fast_tip_major(P) ? P.tip_gene_start[P.T] : 0};
}

template <int T> BIOIK_HD void select_frame(const double (&F)[T][7], int tip, double* f)
{
#pragma unroll
    for(int k = 0; k < 7; k++) f[k] = F[0][k];
#pragma unroll
    for(int t = 1; t < T; t++)
        if(tip == t)
        {
#pragma unroll
            for(int k = 0; k < 7; k++) f[k] = F[t][k];
        }
}

// Goal::evaluate for the link goals, on a frame held in registers (same bodies as goal_value)
BIOIK_HD double link_goal_value(int type, const double* p, const double* f)
{
    switch(type)
    {
    case G_POSITION: return len2(p[0] - f[0], p[1] - f[1], p[2] - f[2]);
    case G_ORIENTATION: return BIOIK_FMIN(qlen2(p[3] - f[3], p[4] - f[4], p[5] - f[5], p[6] - f[6]), qlen2(p[3] + f[3], p[4] + f[4], p[5] + f[5], p[6] + f[6]));
    case G_POSE:
    {
        double e = 0.0;
        e += len2(p[0] - f[0], p[1] - f[1], p[2] - f[2]);
        e += BIOIK_FMIN(qlen2(p[3] - f[3], p[4] - f[4], p[5] - f[5], p[6] - f[6]), qlen2(p[3] + f[3], p[4] + f[4], p[5] + f[5], p[6] + f[6])) * (p[7] * p[7]);
        return e;
    }
    case G_LOOK_AT:
    {
        V3 axis = quat_mul_vec(Q4{f[3], f[4], f[5], f[6]}, V3{p[0], p[1], p[2]});
        double ax = p[3] - f[0], ay = p[4] - f[1], az = p[5] - f[2];
        double sa = 1.0 / BIOIK_SQRT(len2(ax, ay, az));
        ax = ax * sa; ay = ay * sa; az = az * sa;
        double sb = 1.0 / BIOIK_SQRT(len2(axis.x, axis.y, axis.z));
        double bx = axis.x * sb, by = axis.y * sb, bz = axis.z * sb;
        return len2(bx - ax, by - ay, bz - az);
    }
    case G_MAX_DISTANCE:
    {
        double d = BIOIK_FMAX(0.0, BIOIK_SQRT(len2(p[0] - f[0], p[1] - f[1], p[2] - f[2])) - p[3]);
        return d * d;
    }
    case G_MIN_DISTANCE:
    {
        double d = BIOIK_FMAX(0.0, p[3] - BIOIK_SQRT(len2(p[0] - f[0], p[1] - f[1], p[2] - f[2])));
        return d * d;
    }
    case G_LINE:
    {
        double rx = f[0] - p[0], ry = f[1] - p[1], rz = f[2] - p[2];
        double k = p[3] * rx + p[4] * ry + p[5] * rz;
        double qx = f[0] - p[3] * k, qy = f[1] - p[4] * k, qz = f[2] - p[5] * k;
        return len2(qx - p[0], qy - p[1], qz - p[2]);
    }
    case G_PLANE:
    {
        double sd = (f[0] - p[0]) * p[3] + (f[1] - p[1]) * p[4] + (f[2] - p[2]) * p[5];
        return sd * sd;
    }
    case G_SIDE:
    {
        V3 v = quat_mul_vec(Q4{f[3], f[4], f[5], f[6]}, V3{p[0], p[1], p[2]});
        double s = BIOIK_FMAX(0.0, v.x * p[3] + v.y * p[4] + v.z * p[5]);
        return s * s;
    }
    case G_DIRECTION:
    {
        V3 v = quat_mul_vec(Q4{f[3], f[4], f[5], f[6]}, V3{p[0], p[1], p[2]});
        return len2(p[3] - v.x, p[4] - v.y, p[5] - v.z);
    }
    case G_CONE: return cone_goal_value(p, f);
    default: return 0.0;
    }
}

BIOIK_HD bool is_joint_goal(int type) { return type >= G_AVOID_JOINT_LIMITS && type <= G_JOINT_VARIABLE; }

// what one gene adds to a joint-space goal, from its record r = {centre, half span, weight, applies}: the term of
// joint_goal_accumulate, or +0.0 where the goal does not apply to the gene (branch-free: acc + 0.0 == acc, the accumulators
// are never -0).  max(0, y) as a select: fmax(0.0, y) for every y up to the sign of a zero, which the square drops.
BIOIK_HD double joint_record_term(const double* r, bool avoid, double x)
{
    double dd = x - r[0];
    if(avoid)
    {
        const double y = BIOIK_FABS(dd) * 2.0 - r[1];
        dd = bioik_sel_gt0(y, y, 0.0);
    }
    dd *= r[2];
    return bioik_sel_ne0(r[3], dd * dd, 0.0);
}

// one gene's contribution to a joint-space goal (goal_types.h:387-465,494-498), gene order = loop order
BIOIK_HD void joint_goal_accumulate(int type, int var_index, int i, double x, double clip_max, double mid, double halfspan, double vw, double seedv, double p0, double& acc)
{
    switch(type)
    {
    case G_AVOID_JOINT_LIMITS:
        if(clip_max != DBLMAX)
        {
            double d = x - mid;
            d = BIOIK_FMAX(0.0, BIOIK_FABS(d) * 2.0 - halfspan);
            d *= vw;
            acc += d * d;
        }
        break;
    case G_CENTER_JOINTS:
        if(clip_max != DBLMAX)
        {
            double d = x - mid;
            d *= vw;
            acc += d * d;
        }
        break;
    case G_REGULARIZATION:
    {
        double d = x - seedv;
        acc += d * d;
        break;
    }
    case G_MINIMAL_DISPLACEMENT:
    {
        double d = x - seedv;
        d *= vw;
        acc += d * d;
        break;
    }
    case G_JOINT_VARIABLE:
        if(var_index == i)
        {
            double d = p0 - x;
            acc = d * d;
        }
        break;
    default: break;
    }
}

// (over the lanes of `mask`: the whole warp, or the aligned lane group of one task)
// min over the LPT lanes of a task.  With 16 lanes per task the two groups of a warp run the two species of ONE query: they enter,
// loop and leave together, so the reduction is issued warp-wide with a constant full mask - one REDUX per group, back to back.
// (A group mask known only at run time makes the compiler wrap every warp primitive in mask-matching code and run the groups one
// after the other.)
template <int LPT> __device__ __forceinline__ uint32_t group_reduce_min(uint32_t v, unsigned gmask, int lane0)
{
    if(LPT == 32) return __reduce_min_sync(0xffffffffu, v);
    if(LPT == 16)
    {
        const bool upper = lane0 != 0;
        const uint32_t a = __reduce_min_sync(0xffffffffu, upper ? 0xFFFFFFFFu : v);
        const uint32_t b = __reduce_min_sync(0xffffffffu, upper ? v : 0xFFFFFFFFu);
        return upper ? b : a;
    }
    return __reduce_min_sync(gmask, v);
}
// argmin of (fitness key, packed position/child) over the lanes of a task with three reductions: ties -> lowest position (:419-423);
// wkey = the winning key, i.e. the winner's fitness bits
template <int LPT> __device__ __forceinline__ uint32_t fast_warp_argmin(uint64_t key, uint32_t packed, unsigned gmask, int lane0, uint64_t& wkey)
{
    uint32_t hi = (uint32_t)(key >> 32), lo = (uint32_t)key;
    uint32_t mh = group_reduce_min<LPT>(hi, gmask, lane0);
    uint32_t l2 = (hi == mh) ? lo : 0xFFFFFFFFu;
    uint32_t ml = group_reduce_min<LPT>(l2, gmask, lane0);
    uint32_t p2 = (hi == mh && lo == ml) ? packed : 0xFFFFFFFFu;
    wkey = ((uint64_t)mh << 32) | (uint64_t)ml;
    return group_reduce_min<LPT>(p2, gmask, lane0);
}
__device__ __forceinline__ uint64_t fast_fitness_key(double f) { return (f != f) ? 0xFFFFFFFFFFFFFFFEull : (uint64_t)__double_as_longlong(f); }
constexpr uint64_t FAST_KEY_NONE = 0xFFFFFFFFFFFFFFFFull;
__device__ __forceinline__ bool key_less(uint64_t ka, uint32_t pa, uint64_t kb, uint32_t pb) { return ka < kb || (ka == kb && pa < pb); }

#ifndef BIOIK_EVOLVE_WPB
#define BIOIK_EVOLVE_WPB 4 // warps per block of the generation kernels
#endif
#ifndef BIOIK_EVOLVE_MINBLOCKS
#define BIOIK_EVOLVE_MINBLOCKS 4
#endif
constexpr int FAST_MAX_CPL = 8; // population <= 256

// fitness of one genotype under the task's approximator, by a single lane (parents at the start of a step)
template <int T, int GSPEC, bool JOINT>
__device__ __forceinline__ double fast_eval_one(const DProblem& P, int n, const double* x, const double* s_rec, const double* s_delta, const double* s_tip0, const double* s_gp, const double* s_jrec, const double* seed)
{
    double F[T][7];
#pragma unroll
    for(int t = 0; t < T; t++)
#pragma unroll
        for(int j = 0; j < 7; j++) F[t][j] = s_tip0[8 * t + j];
    for(int i = 0; i < n; i++)
    {
        double d = x[i] - s_rec[4 * i + 1];
#pragma unroll
        for(int t = 0; t < T; t++)
        {
            const double* D = s_delta + ((size_t)t * n + i) * 8;
#pragma unroll
            for(int j = 0; j < 7; j++) F[t][j] = BIOIK_FMA(d, D[j], F[t][j]);
        }
    }
    if(GSPEC == 1) return link_goal_value(G_POSE, s_gp, F[0]) * P.goals[0].weight_sq + 0.0;
    double prim = 0.0;
    for(int g = 0; g < P.G; g++)
    {
        const DGoal& gl = P.goals[g];
        if(gl.secondary) continue;
        double v;
        if(JOINT && is_joint_goal(gl.type))
        {
            v = 0.0;
            if(gl.type == G_JOINT_VARIABLE && gl.var_index < 0)
            {
                double dd = s_gp[g * GOAL_NPARAM] - seed[-1 - gl.var_index];
                v = dd * dd;
            }
            else
                for(int i = 0; i < n; i++)
                    joint_goal_accumulate(gl.type, gl.var_index, i, x[i], s_rec[4 * i + 3], s_jrec[4 * i + 0], s_jrec[4 * i + 1], s_jrec[4 * i + 2], s_jrec[4 * i + 3], s_gp[g * GOAL_NPARAM], v);
        }
        else
        {
            double f[7];
            select_frame<T>(F, gl.tip, f);
            v = link_goal_value(gl.type, s_gp + g * GOAL_NPARAM, f);
        }
        prim += v * gl.weight_sq;
    }
    return prim;
}

// the same for any number of tips, goal by goal: a link goal runs the FMA chain of its tip over that tip's gene list (kept
// while consecutive goals read the same tip), so only one tip's frame is live at a time; used by the tip-major kernel form
// (s_delta then holds the delta frames of the (tip, gene) pairs of DProblem::tip_gene, in list order)
template <bool JOINT> __device__ __forceinline__ double fast_eval_one_tips(const DProblem& P, int n, const double* x, const double* s_rec, const double* s_delta, const double* s_tip0, const double* s_gp, const double* s_jrec,
                                                                           const double* seed)
{
    double prim = 0.0;
    double F[7];
    int tip_live = -1;
    for(int g = 0; g < P.G; g++)
    {
        const DGoal& gl = P.goals[g];
        if(gl.secondary) continue;
        double v;
        if(JOINT && is_joint_goal(gl.type))
        {
            v = 0.0;
            if(gl.type == G_JOINT_VARIABLE && gl.var_index < 0)
            {
                double dd = s_gp[g * GOAL_NPARAM] - seed[-1 - gl.var_index];
                v = dd * dd;
            }
            else
                for(int i = 0; i < n; i++)
                    joint_goal_accumulate(gl.type, gl.var_index, i, x[i], s_rec[4 * i + 3], s_jrec[4 * i + 0], s_jrec[4 * i + 1], s_jrec[4 * i + 2], s_jrec[4 * i + 3], s_gp[g * GOAL_NPARAM], v);
        }
        else
        {
            const int t = gl.tip;
            if(t != tip_live)
            {
#pragma unroll
                for(int j = 0; j < 7; j++) F[j] = s_tip0[8 * t + j];
                for(int idx = P.tip_gene_start[t]; idx < P.tip_gene_start[t + 1]; idx++)
                {
                    const int i = P.tip_gene[idx];
                    const double d = x[i] - s_rec[4 * i + 1];
                    const double* D = s_delta + (size_t)idx * 8;
#pragma unroll
                    for(int j = 0; j < 7; j++) F[j] = BIOIK_FMA(d, D[j], F[j]);
                }
                tip_live = t;
            }
            v = link_goal_value(gl.type, s_gp + g * GOAL_NPARAM, F);
        }
        prim += v * gl.weight_sq;
    }
    return prim;
}

// T = tips, CH = children evaluated together per lane (register block),
// GSPEC = 1: the problem is exactly one primary PoseGoal (the plugin's default goal for a one-tip group);
// JOINT: joint-space goals present (accumulated in the gene loop)
// NG: gene count as a compile-time constant (0 = P.n at run time): the gene loop unrolls, its pointer bumps fold into immediates
// TM (tip-major form, T must be 1): any number of tips P.T, one tip's frame accumulators at a time over that tip's gene list
// LPT (lanes per task): 32 = one warp per task; 16 / 8 = two / four tasks per warp, each lane then owns 8 / 16 children.  The
// per-child work is lane-efficient either way, but the per-generation overhead (tables, the two argmin reductions, winner
// re-derivation: a large share of the instructions at LPT 32) is issued once per WARP, i.e. shared by the tasks of the warp.
// The body of the generation kernel for ONE task = (query, species slot): `generations` x {reproduce, phenotype, fitness, selection}
// of step `step`, run by the LPT lanes `gmask` of a warp (lane = index inside that group, lane0 = its first warp lane) on the
// shared-memory block W (FastSmem::total() doubles).  Called by k_evolve_fast (one launch per step) and by the persistent
// solve kernel (bioik_persist.cuh), which keeps warps resident and feeds them (query, step) items from a queue.
template <int T, int CH, int GSPEC, bool JOINT, int NG, bool TM, int LPT>
__device__ __forceinline__ void evolve_fast_task(const DProblem& P, const DState& S, int step, const double* __restrict__ mtab, double* W, int task, int lane, int lane0, unsigned gmask)
{
    static_assert(LPT == 32 || (LPT == 16 || LPT == 8) && !TM && GSPEC == 1 && !JOINT, "lane groups are instantiated for the single-pose problem only");
    // the single-pose problem with a compile-time gene count (NG <= 8 genes sit in the first lanes of a lane group; with 16 lanes per
    // task both groups of a warp hold the two species of one query, so they enter and leave together and warp-wide votes are safe)
    constexpr bool LEAN = NG != 0 && NG <= 8 && GSPEC == 1 && !JOINT && !TM && (LPT == 16 || LPT == 32);
    // mask of the warp-level primitives: with 16 lanes per task both groups of the warp are always here together (above), so they
    // are issued warp-wide with a constant mask; lane indices passed to shuffles are warp lanes (lane0 + ...) either way
    const unsigned smask = (LPT == 32 || LPT == 16) ? 0xffffffffu : gmask;
    if(task >= S.B * 2) return;
    const int q = task >> 1, slot = task & 1;
    // asked first, acted on after the staging loads below are in flight: the flags it reads are another round trip to L2
    const bool finished = run_done(S, q, step);
    const bool has_sec = LEAN ? false : P.has_secondary != 0; // (a single primary PoseGoal has no secondary goals: compile-time for the LEAN forms)
    const int n = NG ? NG : P.n, C = S.C, G = P.G;
    const int R = mtab_row(C);
    const int nchunks = R / (LPT * CH); // R is a power of two >= LPT * CH (select_evolve_fast)
    // joint-space goals in goal order: slot j of the accumulators = the j-th of them; avoid_j = AvoidJointLimitsGoal
    int nj = 0;
    bool jq_avoid[FAST_MAX_JOINT_GOALS];
#pragma unroll
    for(int j = 0; j < FAST_MAX_JOINT_GOALS; j++) jq_avoid[j] = false;
    if(JOINT)
        for(int g = 0; g < G; g++)
            if(is_joint_goal(P.goals[g].type) && nj < FAST_MAX_JOINT_GOALS)
            {
#pragma unroll
                for(int j = 0; j < FAST_MAX_JOINT_GOALS; j++)
                    if(j == nj) jq_avoid[j] = P.goals[g].type == G_AVOID_JOINT_LIMITS;
                nj++;
            }

    FastSmem L{n, TM ? P.T : T, G, JOINT ? P.n_joint_goals : 0, has_sec ? 0 : 1, TM ? P.tip_gene_start[P.T] : 0};
    const int TT = TM ? P.T : T; // tips of the problem
    double *s_rec = W + L.off_rec(), *s_term = W + L.off_term(), *s_delta = W + L.off_delta(), *s_par = W + L.off_par(), *s_pg = W + L.off_pg();
    double *s_tip0 = W + L.off_tip0(), *s_gp = W + L.off_gp(), *s_jrec = W + L.off_jrec(), *s_jq = W + L.off_jq(), *s_fit = W + L.off_fit(), *s_sf = W + L.off_sf();
    double *s_prec = W + L.off_prec(), *s_pterm = W + L.off_pterm();
    const double* seed = S.seeds + (size_t)q * P.n_vars;

    // ---- stage the task -------------------------------------------------------------------
    if(TM)
    {
        // only the (tip, gene) pairs with a delta frame that can be non-zero, in the order the chains read them
        for(int k = lane; k < L.pairs * 7; k += LPT)
        {
            const int idx = k / 7, c7 = k - idx * 7;
            int t = 0;
            while(P.tip_gene_start[t + 1] <= idx) t++;
            s_delta[idx * 8 + c7] = S.delta[(size_t)task * TT * n * 7 + ((size_t)t * n + P.tip_gene[idx]) * 7 + c7];
        }
        for(int idx = lane; idx < L.pairs; idx += LPT) s_delta[idx * 8 + 7] = __longlong_as_double((long long)P.tip_gene[idx] * mtab_row(S.C));
    }
    else
        for(int k = lane; k < TT * n * 7; k += LPT)
        {
            int ti = k / 7, c7 = k - ti * 7;
            s_delta[ti * 8 + c7] = S.delta[(size_t)task * TT * n * 7 + k];
        }
    for(int k = lane; k < TT * 7; k += LPT) s_tip0[(k / 7) * 8 + (k % 7)] = S.tip0[(size_t)task * TT * 7 + k];
    for(int i = lane; i < n; i += LPT)
    {
        const DGene& Gn = P.genes[i];
        s_rec[4 * i + 1] = S.base[(size_t)task * n + i];
        s_rec[4 * i + 2] = Gn.clip_min;
        s_rec[4 * i + 3] = Gn.clip_max;
        s_par[0 * n + i] = S.genes[((size_t)task * 2 + 0) * n + i];
        s_par[1 * n + i] = S.genes[((size_t)task * 2 + 1) * n + i];
        s_par[2 * n + i] = S.grads[((size_t)task * 2 + 0) * n + i];
        s_par[3 * n + i] = S.grads[((size_t)task * 2 + 1) * n + i];
        if(JOINT)
        {
            s_jrec[4 * i + 0] = (Gn.vmin + Gn.vmax) * 0.5;
            s_jrec[4 * i + 1] = Gn.span * 0.5;
            s_jrec[4 * i + 2] = Gn.vel_weight;
            s_jrec[4 * i + 3] = seed[Gn.var];
        }
    }
    for(int k = lane; k < G * GOAL_NPARAM; k += LPT) s_gp[k] = S.goal_params[(size_t)q * G * GOAL_NPARAM + k];
    if(finished) return; // the run is over (all lanes of the task - with 16 lanes per task: of the warp - agree); nothing was written
    __syncwarp(smask);
    if(TM) // the per-task part of the pair records: base and clip limits of the pair's gene
        for(int idx = lane; idx < L.pairs; idx += LPT)
        {
            const int i = P.tip_gene[idx];
            s_prec[4 * idx + 1] = s_rec[4 * i + 1];
            s_prec[4 * idx + 2] = s_rec[4 * i + 2];
            s_prec[4 * idx + 3] = s_rec[4 * i + 3];
        }
    if(JOINT)
    {
        // One record per (joint-space goal, gene): every such goal adds ((x - centre) [-> max(0, |.| * 2 - half span)]) * weight,
        // squared, for the genes it applies to (goal_types.h:387-465,494-498).  RegularizationGoal and JointVariableGoal have
        // no weight factor: * 1.0 is exact; JointVariableGoal's (p0 - x)^2 == (x - p0)^2 bit for bit and 0.0 + that == that.
        int j = 0;
        for(int g = 0; g < G; g++)
        {
            const DGoal& gl = P.goals[g];
            if(!is_joint_goal(gl.type) || j >= FAST_MAX_JOINT_GOALS) continue;
            for(int i = lane; i < n; i += LPT)
            {
                const DGene& Gn = P.genes[i];
                double c = 0.0, w = 1.0, on = 1.0;
                const double mid = (Gn.vmin + Gn.vmax) * 0.5, seedv = seed[Gn.var];
                switch(gl.type)
                {
                case G_AVOID_JOINT_LIMITS: c = mid, w = Gn.vel_weight, on = Gn.clip_max != DBLMAX ? 1.0 : 0.0; break;
                case G_CENTER_JOINTS: c = mid, w = Gn.vel_weight, on = Gn.clip_max != DBLMAX ? 1.0 : 0.0; break;
                case G_REGULARIZATION: c = seedv; break;
                case G_MINIMAL_DISPLACEMENT: c = seedv, w = Gn.vel_weight; break;
                default: c = s_gp[g * GOAL_NPARAM], on = gl.var_index == i ? 1.0 : 0.0; break; // G_JOINT_VARIABLE
                }
                double* r = s_jq + ((size_t)j * n + i) * 4;
                r[0] = c, r[1] = Gn.span * 0.5, r[2] = w, r[3] = on;
            }
            j++;
        }
        __syncwarp(smask);
    }

    // Fitness of the two parents under this step's approximator.  Within a step the parents of generation
    // g+1 are the winners of generation g, whose fitness (same genes, same operations) is already known,
    // so children[0..1] (:381-388,:401-407) are evaluated once here and carried in registers afterwards.
    double pf = 0.0;
    if(lane < 2) pf = TM ? fast_eval_one_tips<JOINT>(P, n, s_par + lane * n, s_rec, s_delta, s_tip0, s_gp, s_jrec, seed) : fast_eval_one<T, GSPEC, JOINT>(P, n, s_par + lane * n, s_rec, s_delta, s_tip0, s_gp, s_jrec, seed);
    double f_par0 = __shfl_sync(smask, pf, lane0 + 0), f_par1 = __shfl_sync(smask, pf, lane0 + 1);

    // clamp elision (below): the largest mutation of this lane's gene, hoisted out of the generation loop
    double lean_reach = 0.0;
    if(LEAN && lane < n) lean_reach = S.gauss_absmax * (1.0 / 256.0) * P.genes[lane].span;
    int cur = 0;                 // parent buffer in use
    const int parity = lane & 1; // child slot c = j + 2 is even <=> lane is even
    // EARLY: the first mutation-table row of a chunk is requested while the previous chunk's fitness (or the previous generation's
    // selection) is still being worked on, so its latency is off the chunk's dependent chain
    constexpr bool EARLY = BIOIK_EVOLVE_EARLYROW && LEAN;
    double m_early[EARLY ? CH : 1];
    if(EARLY)
    {
        const double* mt0 = mtab + (size_t)((stream_step(S, q, step) * 2 + slot) * S.gens) * n * R;
#pragma unroll
        for(int k = 0; k < CH; k++) m_early[k] = BIOIK_LDG(mt0 + lane + LPT * k);
    }
    const double wsq0 = P.goals[0].weight_sq;

    for(int gen = 0; gen < S.gens; gen++)
    {
        const int call = (stream_step(S, q, step) * 2 + slot) * S.gens + gen;
        const double* mt = mtab + (size_t)call * n * R;
        const int child_count = has_sec ? S.ccount[((size_t)q * 2 + slot) * S.gens + gen] : C;
        double* par = s_par + cur * 4 * n;
        const double *p_g0 = par, *p_g1 = par + n, *p_gr0 = par + 2 * n, *p_gr1 = par + 3 * n;

        // per-generation warp-uniform tables: pg = mix(gr0, gr1, fmix), term = pg * gradient_factor  (:268-269,:294-295)
        bool gene_safe = false;
        for(int i = lane; i < n; i += LPT)
        {
            double a = p_gr0[i], b = p_gr1[i];
            double pge = mix(a, b, 0.2); // child_index even: fmix = 1 * 0.2
            double pgo = mix(a, b, 0.0); // child_index odd:  fmix = 0 * 0.2
            s_pg[i] = pge;
            s_pg[n + i] = pgo;
            s_term[6 * i + 0] = pge * 0.0;
            s_term[6 * i + 1] = pge * 1.0;
            s_term[6 * i + 2] = pge * 2.0;
            s_term[6 * i + 3] = pgo * 0.0;
            s_term[6 * i + 4] = pgo * 1.0;
            s_term[6 * i + 5] = pgo * 2.0;
            s_rec[4 * i + 0] = p_g0[i];
            if(LEAN)
            {
                // Clamp elision: every child gene of this generation is fl(fl(g0 + m) + t) with |m| <= gauss_absmax * 2^-8 * span
                // (mutation_rate <= 2^15 / 2^23, :265,:290-293) and t in {0, pg, 2 pg} (:294-296).  If g0 keeps that distance (plus
                // rounding slack) from both clip limits, clamp() returns its argument for all children and is skipped for the gene.
                const double g0 = p_g0[i];
                const double e = (lean_reach + 2.0 * BIOIK_FMAX(BIOIK_FABS(pge), BIOIK_FABS(pgo))) * 1.000001; // i == lane: n <= 8 < LPT
                const double slack = e + 1e-15 * (BIOIK_FABS(g0) + e);
#ifndef BIOIK_X_NOELIDE
                gene_safe = (g0 - slack > s_rec[4 * i + 2]) && (g0 + slack < s_rec[4 * i + 3]); // false for NaN: the clamp stays
#endif
            }
        }
        unsigned unclamped = 0u; // bit i: gene i needs no clamp in this generation, for every task of the warp (warp-uniform)
        if(LEAN)
        {
            const unsigned safe = __ballot_sync(0xffffffffu, gene_safe);
            unclamped = LPT == 16 ? (safe & (safe >> 16)) : safe; // lanes 0..NG-1 of every lane group hold the genes
        }
        __syncwarp(smask);
        if(TM)
        {
            // the per-generation part of the pair records: parent gene and the six gradient terms of the pair's gene
            for(int idx = lane; idx < L.pairs; idx += LPT)
            {
                const int i = P.tip_gene[idx];
                s_prec[4 * idx + 0] = s_rec[4 * i + 0];
#pragma unroll
                for(int c = 0; c < 6; c++) s_pterm[6 * idx + c] = s_term[6 * i + c];
            }
            __syncwarp(smask);
        }

        // this lane's two best children so far: (key, packed = position * 512 + child)
        uint64_t k1 = FAST_KEY_NONE, k2 = FAST_KEY_NONE;
        uint32_t q1 = 0xFFFFFFFFu, q2 = 0xFFFFFFFFu;
        double b1 = 0.0, b2 = 0.0; // fitness values of q1 / q2 while no pre-selection is active

        for(int chunk = 0; chunk < nchunks; chunk++)
        {
            const int jbase = lane + LPT * CH * chunk; // child slot c = j + 2
            double F[CH][T][7];
            double acc[JOINT ? CH : 1][FAST_MAX_JOINT_GOALS];
            const double* tp[CH]; // term column of each child: fmix class x gradient_factor (c % 3)
#pragma unroll
            for(int k = 0; k < CH; k++)
            {
                int c = jbase + LPT * k + 2;
                tp[k] = s_term + (parity ? 3 : 0) + (c % 3);
                if(JOINT)
#pragma unroll
                    for(int j = 0; j < FAST_MAX_JOINT_GOALS; j++) acc[k][j] = 0.0;
            }
            double tm_prim[TM ? CH : 1], tm_sec[TM ? CH : 1];
            if(TM)
            {
                // ---- tip-major form: a tip's frames are the FMA chain over the genes that can move it (ascending = the order of the
                // gene-major chain restricted to that tip; the skipped genes have an all-zero delta frame, fma(d, 0, F) == F), run
                // when the first goal of that tip comes up in goal order.  Only 7 accumulators per child are live, whatever the
                // number of tips.
                auto gene_value = [&](int i, int k) { // :293-297 for child k of this lane
                    double gene = s_rec[4 * i + 0];
                    gene += BIOIK_LDG(mt + (size_t)i * R + jbase + LPT * k); // gene += r * f
                    gene += tp[k][6 * i];                                   // gene += gradient
                    return clampd(gene, s_rec[4 * i + 2], s_rec[4 * i + 3]);
                };
                if(JOINT)
                    for(int i = 0; i < n; i++)
                    {
                        double x[CH];
#pragma unroll
                        for(int k = 0; k < CH; k++) x[k] = gene_value(i, k);
#pragma unroll
                        for(int j = 0; j < FAST_MAX_JOINT_GOALS; j++)
                            if(j < nj)
                            {
                                const double* r = s_jq + ((size_t)j * n + i) * 4;
#pragma unroll
                                for(int k = 0; k < CH; k++) acc[k][j] += joint_record_term(r, jq_avoid[j], x[k]);
                            }
                    }
                // weighted sums in goal order (src/problem.cpp:251-257): a link goal finds its tip's frames in F (kept while
                // consecutive goals read the same tip), a joint-space goal its accumulator
                int tip_live = -1, jn = 0;
#pragma unroll
                for(int k = 0; k < CH; k++) tm_prim[k] = 0.0, tm_sec[k] = 0.0;
                for(int g = 0; g < G; g++)
                {
                    const DGoal& gl = P.goals[g];
                    double v[CH];
                    if(JOINT && is_joint_goal(gl.type))
                    {
#pragma unroll
                        for(int k = 0; k < CH; k++)
                        {
                            v[k] = 0.0;
#pragma unroll
                            for(int j = 0; j < FAST_MAX_JOINT_GOALS; j++)
                                if(j == jn) v[k] = acc[k][j];
                            if(gl.type == G_JOINT_VARIABLE && gl.var_index < 0)
                            {
                                double dd = s_gp[g * GOAL_NPARAM] - seed[-1 - gl.var_index];
                                v[k] = dd * dd;
                            }
                        }
                        jn++;
                    }
                    else if(gl.secondary)
                    {
                        // secondary goals see null_tip_frames (identity), src/ik_base.h:163
                        const double f[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0};
                        const double vv = link_goal_value(gl.type, s_gp + g * GOAL_NPARAM, f);
#pragma unroll
                        for(int k = 0; k < CH; k++) v[k] = vv;
                    }
                    else
                    {
                        const int t = gl.tip;
                        if(t != tip_live)
                        {
                            tip_live = t;
#pragma unroll
                            for(int k = 0; k < CH; k++)
#pragma unroll
                                for(int j = 0; j < 7; j++) F[k][0][j] = s_tip0[8 * t + j];
                            int idx = P.tip_gene_start[t];
                            const int i1 = P.tip_gene_start[t + 1];
                            // the chain walks the pair records (s_prec, s_delta, s_pterm are in pair order): pointer bumps, no indexing by
                            // gene; mutation terms are fetched one list entry ahead of their use, from the table offset in the pad slot
                            // of the pair's delta frame
                            const double* pr = s_prec + 4 * idx;
                            const double* D = s_delta + 8 * idx;
                            const double* pt[CH];
#pragma unroll
                            for(int k = 0; k < CH; k++) pt[k] = s_pterm + 6 * idx + (tp[k] - s_term);
                            const double* mb = mt + jbase;
                            double m[CH];
                            {
                                const long long off = idx < i1 ? __double_as_longlong(D[7]) : 0ll;
#pragma unroll
                                for(int k = 0; k < CH; k++) m[k] = BIOIK_LDG(mb + off + LPT * k);
                            }
#pragma unroll 2
                            for(; idx < i1; idx++)
                            {
                                const long long offn = __double_as_longlong(idx + 1 < i1 ? D[8 + 7] : D[7]);
                                double mnext[CH];
#pragma unroll
                                for(int k = 0; k < CH; k++) mnext[k] = BIOIK_LDG(mb + offn + LPT * k);
                                const double g0 = pr[0], base = pr[1], lo = pr[2], hi = pr[3];
                                double Dv[7];
#pragma unroll
                                for(int j = 0; j < 7; j++) Dv[j] = D[j];
#pragma unroll
                                for(int k = 0; k < CH; k++)
                                {
                                    double gene = g0;
                                    gene += m[k];     // gene += r * f      (:293)
                                    gene += pt[k][0]; // gene += gradient   (:296)
                                    gene = clampd(gene, lo, hi);
                                    const double d = gene - base; // :1086
#pragma unroll
                                    for(int j = 0; j < 7; j++) F[k][0][j] = BIOIK_FMA(d, Dv[j], F[k][0][j]);
                                    m[k] = mnext[k];
                                    pt[k] += 6;
                                }
                                pr += 4;
                                D += 8;
                            }
                        }
#pragma unroll
                        for(int k = 0; k < CH; k++) v[k] = link_goal_value(gl.type, s_gp + g * GOAL_NPARAM, F[k][0]);
                    }
#pragma unroll
                    for(int k = 0; k < CH; k++)
                    {
                        if(gl.secondary)
                            tm_sec[k] += v[k] * gl.weight_sq;
                        else
                            tm_prim[k] += v[k] * gl.weight_sq;
                    }
                }
            }
            else
            {
                const double* mp = mt + jbase;
                const double* rp = s_rec;
                const double* dp = s_delta;

                // mutation terms are fetched one gene ahead of their use (L1/L2 latency off the dependent chain)
                // (two register buffers used alternately: no register rotation in the loop)
                double mA[CH], mB[CH];
    #pragma unroll
                for(int k = 0; k < CH; k++) mA[k] = EARLY ? m_early[k] : BIOIK_LDG(mp + LPT * k);

                // one gene of all CH children; FIRST = the accumulators start from the base tip frames (no copy)
                auto gene_step = [&](auto first_tag, int i, const double (&m)[CH], double (&mnext)[CH]) {
                    constexpr bool FIRST = decltype(first_tag)::value;
                    const double g0 = rp[0], base = rp[1], lo = rp[2], hi = rp[3];
                    double d[CH], x[CH];
                    mp += R;
                    if(i + 1 < n)
                    {
    #pragma unroll
                        for(int k = 0; k < CH; k++) mnext[k] = BIOIK_LDG(mp + LPT * k);
                    }
    #pragma unroll
                    for(int k = 0; k < CH; k++)
                    {
                        double gene = g0;
                        gene += m[k];                // gene += r * f      (:293)
                        gene += tp[k][0];            // gene += gradient   (:296)
                        x[k] = gene;
                    }
                    if(!(LEAN && ((unclamped >> i) & 1u))) // :297 (warp-uniform: skipped where clamp() is the identity for every child)
                    {
#pragma unroll
                        for(int k = 0; k < CH; k++) x[k] = clampd(x[k], lo, hi);
                    }
#pragma unroll
                    for(int k = 0; k < CH; k++)
                    {
                        const double gene = x[k];
                        d[k] = gene - base; // :1086
                        tp[k] += 6;
                    }
                    rp += 4;
                    const int tmask = (T == 1) ? 1 : P.genes[i].tipmask; // tips this gene can move (structural); others have an all-zero delta frame
    #pragma unroll
                    for(int t = 0; t < T; t++)
                    {
                        const bool on = (tmask >> t) & 1;
                        if(!on && !FIRST) continue; // fma(d, 0, F) == F
                        const double* D = dp + (size_t)t * n * 8;
                        double Dv[7];
    #pragma unroll
                        for(int j = 0; j < 7; j++) Dv[j] = on ? D[j] : 0.0;
    #pragma unroll
                        for(int k = 0; k < CH; k++)
    #pragma unroll
                            for(int j = 0; j < 7; j++) F[k][t][j] = BIOIK_FMA(d[k], Dv[j], FIRST ? s_tip0[8 * t + j] : F[k][t][j]);
                    }
                    dp += 8;
                    if(JOINT)
                    {
    #pragma unroll
                        for(int j = 0; j < FAST_MAX_JOINT_GOALS; j++)
                            if(j < nj)
                            {
                                const double* r = s_jq + ((size_t)j * n + i) * 4;
    #pragma unroll
                                for(int k = 0; k < CH; k++) acc[k][j] += joint_record_term(r, jq_avoid[j], x[k]);
                            }
                    }
                };
                gene_step(std::true_type{}, 0, mA, mB);
                if(NG)
                {
    #pragma unroll
                    for(int i = 1; i < NG; i++)
                    {
                        if(i & 1)
                            gene_step(std::false_type{}, i, mB, mA);
                        else
                            gene_step(std::false_type{}, i, mA, mB);
                    }
                }
                else
                {
                    int i = 1;
    #pragma unroll 1
                    for(; i + 1 < n; i += 2)
                    {
                        gene_step(std::false_type{}, i, mB, mA);
                        gene_step(std::false_type{}, i + 1, mA, mB);
                    }
                    if(i < n) gene_step(std::false_type{}, i, mB, mA);
                }
                if(EARLY)
                {
                    // next chunk of this generation, else the first chunk of the next generation (the table rows of the call after
                    // the last one of the step exist: the schedule is sized for the whole solve; beyond it the request is skipped)
                    const bool more = chunk + 1 < nchunks;
                    const double* nx = more ? mt + jbase + LPT * CH : mt + (size_t)n * R + lane;
                    if(more || gen + 1 < S.gens)
                    {
#pragma unroll
                        for(int k = 0; k < CH; k++) m_early[k] = BIOIK_LDG(nx + LPT * k);
                    }
                }
            }

            // fitness: weighted sum in goal order (src/problem.cpp:251-257)
#pragma unroll
            for(int k = 0; k < CH; k++)
            {
                const int c = jbase + LPT * k + 2;
                double prim = 0.0, sec = 0.0;
                if(LEAN)
                {
                    // PoseGoal::evaluate * weight_sq (goal_types.h:149-180, problem.cpp:251-257) without the additions to a zero
                    // accumulator (exact: every summand is >= +0 or NaN) and with fmin as a select (both norms are NaN together)
                    const double* f = F[k][0];
                    const double e_pos = len2(s_gp[0] - f[0], s_gp[1] - f[1], s_gp[2] - f[2]);
                    const double qm = qlen2(s_gp[3] - f[3], s_gp[4] - f[4], s_gp[5] - f[5], s_gp[6] - f[6]);
                    const double qp = qlen2(s_gp[3] + f[3], s_gp[4] + f[4], s_gp[5] + f[5], s_gp[6] + f[6]);
                    prim = (e_pos + (qm < qp ? qm : qp) * (s_gp[7] * s_gp[7])) * wsq0;
                    // running top-2 of this lane on the integer keys of the fitness (the order the selection uses, NaN last): a lane
                    // meets its children in increasing position order, so the strict < keeps the earlier one on ties - branch-free
                    const uint64_t key = c < C ? fast_fitness_key(prim) : FAST_KEY_NONE;
                    const uint32_t pk = (uint32_t)c * 512u + (uint32_t)c;
                    const bool lt1 = key < k1, lt2 = key < k2;
                    k2 = lt1 ? k1 : (lt2 ? key : k2);
                    q2 = lt1 ? q1 : (lt2 ? pk : q2);
                    k1 = lt1 ? key : k1;
                    q1 = lt1 ? pk : q1;
                    continue;
                }
                if(TM)
                    prim = tm_prim[k], sec = tm_sec[k];
                else if(GSPEC == 1)
                    prim += link_goal_value(G_POSE, s_gp, F[k][0]) * wsq0;
                else
                {
                    int jn = 0;
                    for(int g = 0; g < G; g++)
                    {
                        const DGoal& gl = P.goals[g];
                        double v;
                        if(JOINT && is_joint_goal(gl.type))
                        {
                            v = 0.0;
#pragma unroll
                            for(int j = 0; j < FAST_MAX_JOINT_GOALS; j++)
                                if(j == jn) v = acc[k][j];
                            if(gl.type == G_JOINT_VARIABLE && gl.var_index < 0)
                            {
                                double dd = s_gp[g * GOAL_NPARAM] - seed[-1 - gl.var_index];
                                v = dd * dd;
                            }
                            jn++;
                        }
                        else
                        {
                            {
                                double f[7];
                                select_frame<T>(F[k], gl.secondary ? 0 : gl.tip, f);
                                if(gl.secondary)
                                {
                                    // secondary goals see null_tip_frames (identity), src/ik_base.h:163
                                    f[0] = f[1] = f[2] = f[3] = f[4] = f[5] = 0.0;
                                    f[6] = 1.0;
                                }
                                v = link_goal_value(gl.type, s_gp + g * GOAL_NPARAM, f);
                            }
                        }
                        if(gl.secondary)
                            sec += v * gl.weight_sq;
                        else
                            prim += v * gl.weight_sq;
                    }
                }
                if(has_sec)
                {
                    if(c < C)
                    {
                        s_fit[c] = prim;
                        s_sf[c] = sec;
                    }
                }
                else if(c < C)
                {
                    // running top-2 of this lane on the fitness VALUES; position == child slot without pre-selection.
                    // Order = order of the integer keys: any number beats a NaN, and since a lane meets its children in
                    // increasing position order ties keep the earlier one (strict <).
                    const uint32_t pk = (uint32_t)c * 512u + (uint32_t)c;
                    const bool ok = prim == prim;
                    if(q1 == 0xFFFFFFFFu || prim < b1 || (b1 != b1 && ok))
                    {
                        b2 = b1; q2 = q1;
                        b1 = prim; q1 = pk;
                    }
                    else if(q2 == 0xFFFFFFFFu || prim < b2 || (b2 != b2 && ok))
                    {
                        b2 = prim; q2 = pk;
                    }
                }
            }
        }
        if(!has_sec && !LEAN)
        {
            k1 = q1 == 0xFFFFFFFFu ? FAST_KEY_NONE : fast_fitness_key(b1);
            k2 = q2 == 0xFFFFFFFFu ? FAST_KEY_NONE : fast_fitness_key(b2);
        }

        if(has_sec)
        {
            // pre-selection (:366-378): position = 2 + stable rank of the secondary fitness; only the first
            // child_count positions take part in the selection
            __syncwarp(smask);
            // the lane's children c0, c0 + 32, ... (c0 = its first child slot >= 2), all NB of them together: one broadcast read of
            // every other child's secondary fitness serves NB ranks.
            // Fast pass: rank' = how many children have a strictly smaller secondary fitness (one DSETP per pair).  rank' is the
            // stable rank unless two children tie or one of the values is a NaN, and in both cases two children share a rank'
            // (equal values count the same set; a NaN counts nobody, like the smallest value) - so the ranks the warp found are
            // collected in a bitmap, and only if fewer distinct ranks than children turn up the exact pass (ties broken by child
            // slot: lt | (eq & before)) runs.  Both passes give the reference's order; the exact one is the rare path.
            const int c0 = lane < 2 ? lane + 32 : lane;
            auto rank_all = [&](auto nb_tag) {
                constexpr int NB = decltype(nb_tag)::value;
                double mine[NB];
                int rank[NB];
#pragma unroll
                for(int j = 0; j < NB; j++)
                {
                    const int c = c0 + 32 * j;
                    mine[j] = c < C ? s_sf[c] : 0.0;
                    rank[j] = 0;
                }
                for(int o = 2; o < C; o++)
                {
                    const double other = s_sf[o];
#pragma unroll
                    for(int j = 0; j < NB; j++) rank[j] += other < mine[j] ? 1 : 0;
                }
                // distinct ranks of the task: bit r of the bitmap = some child has rank' r (ranks are < C - 2 <= 32 * NB)
                int distinct = 0;
#pragma unroll
                for(int w = 0; w < NB; w++)
                {
                    unsigned bits = 0u;
#pragma unroll
                    for(int j = 0; j < NB; j++)
                        if(c0 + 32 * j < C && (rank[j] >> 5) == w) bits |= 1u << (rank[j] & 31);
                    distinct += __popc(__reduce_or_sync(gmask, bits));
                }
                if(distinct != C - 2) // warp-uniform
                {
#pragma unroll
                    for(int j = 0; j < NB; j++) rank[j] = 0;
                    for(int o = 2; o < C; o++)
                    {
                        const double other = s_sf[o];
#pragma unroll
                        for(int j = 0; j < NB; j++)
                        {
                            // no short-circuit: evaluated as predicate logic, not as data-dependent (divergent) branches
                            const int lt = other < mine[j] ? 1 : 0, eq = other == mine[j] ? 1 : 0, before = o < c0 + 32 * j ? 1 : 0;
                            rank[j] += lt | (eq & before);
                        }
                    }
                }
#pragma unroll
                for(int j = 0; j < NB; j++)
                {
                    const int c = c0 + 32 * j;
                    if(c >= C) continue;
                    if(2 + rank[j] >= child_count) continue;
                    uint64_t kk = fast_fitness_key(s_fit[c]);
                    uint32_t pk = (uint32_t)(2 + rank[j]) * 512u + (uint32_t)c;
                    if(key_less(kk, pk, k1, q1))
                    {
                        k2 = k1; q2 = q1;
                        k1 = kk; q1 = pk;
                    }
                    else if(key_less(kk, pk, k2, q2))
                    {
                        k2 = kk; q2 = pk;
                    }
                }
            };
            const int per_lane = (C - 2 + 31) / 32; // children of the busiest lane (C <= 256: at most 8)
            if(per_lane <= 2)
                rank_all(std::integral_constant<int, 2>{});
            else if(per_lane <= 4)
                rank_all(std::integral_constant<int, 4>{});
            else
                rank_all(std::integral_constant<int, 8>{});
        }

        // ---- selection (:410-431): two strict-< scans in position order ----------------------------------
        // candidates: parent 0 at position 0, parent 1 at position 1 (cached fitness), each lane's best child
        uint32_t w1;
        uint64_t wkey1, wkey2; // keys of the two winners = their fitness bits
        {
            uint64_t kk = k1;
            uint32_t pk = q1;
            uint64_t kp0 = fast_fitness_key(f_par0), kp1 = fast_fitness_key(f_par1);
            if(lane == 0 && key_less(kp0, 0u, kk, pk)) { kk = kp0; pk = 0u; }
            if(lane == 1 && key_less(kp1, 512u + 1u, kk, pk)) { kk = kp1; pk = 512u + 1u; }
            w1 = fast_warp_argmin<LPT>(kk, pk, gmask, lane0, wkey1);
            if(f_par0 != f_par0) w1 = 0u; // position 0 holds a NaN: `f < fmin` never fires (:418-422)
        }
        const uint32_t w1_pos = w1 >> 9, w1_child = w1 & 511u;
        uint32_t w2;
        {
            // drop winner 1; after the swap (:424) the element that was at position 0 sits at position w1_pos
            uint64_t kk = k1;
            uint32_t pk = q1;
            if(pk == w1) { kk = k2; pk = q2; }
            uint64_t kp0 = fast_fitness_key(f_par0), kp1 = fast_fitness_key(f_par1);
            if(lane == 0 && w1_child != 0u && key_less(kp0, w1_pos * 512u, kk, pk)) { kk = kp0; pk = w1_pos * 512u; }
            if(lane == 1 && w1_child != 1u && key_less(kp1, 512u + 1u, kk, pk)) { kk = kp1; pk = 512u + 1u; }
            w2 = fast_warp_argmin<LPT>(kk, pk, gmask, lane0, wkey2);
            // the scan starts at position 1: its occupant wins if its fitness is NaN
            uint32_t occ1 = (w1_pos == 1u) ? 0u : 1u;
            double f_occ1 = occ1 == 0u ? f_par0 : f_par1;
            if(f_occ1 != f_occ1) w2 = occ1 | (1u << 9);
        }
        const uint32_t w2_child = w2 & 511u;

        // fitness of the winners = parents' fitness of the next generation: a child's is the key its argmin returned (the key of a
        // number is its bit pattern; a NaN comes back as a NaN), parents keep their cached value
        {
            const double nf0 = w1_child >= 2u ? __longlong_as_double((long long)wkey1) : (w1_child == 0u ? f_par0 : f_par1);
            const double nf1 = w2_child >= 2u ? __longlong_as_double((long long)wkey2) : (w2_child == 0u ? f_par0 : f_par1);
            f_par0 = nf0;
            f_par1 = nf1;
        }

        // ---- new parents into the other buffer: lane i re-derives gene i of both winners --------------
        double* nxt = s_par + (cur ^ 1) * 4 * n;
        {
            const int wc1 = (int)w1_child, wc2 = (int)w2_child;
            for(int i = lane; i < n; i += LPT)
            {
                const double g0 = p_g0[i], lo = s_rec[4 * i + 2], hi = s_rec[4 * i + 3];
#pragma unroll
                for(int w = 0; w < 2; w++)
                {
                    const int wc = w ? wc2 : wc1;
                    double gene, gr;
                    if(wc < 2)
                    {
                        gene = wc == 0 ? g0 : p_g1[i];
                        gr = wc == 0 ? p_gr0[i] : p_gr1[i];
                    }
                    else
                    {
                        const int wpar = wc & 1; // 1 = odd child
                        gene = g0;
                        gene += BIOIK_LDG(mt + (size_t)i * R + (wc - 2));
                        gene += s_term[6 * i + (wpar ? 3 : 0) + (wc % 3)];
                        gene = clampd(gene, lo, hi);
                        gr = mix(s_pg[wpar * n + i], gene - g0, 0.3); // :299
                    }
                    nxt[w * n + i] = gene;      // genes of individuals[w]
                    nxt[(2 + w) * n + i] = gr;  // gradients
                }
            }
        }
        __syncwarp(smask);
        cur ^= 1;
    }

    double* par = s_par + cur * 4 * n;
    for(int i = lane; i < n; i += LPT)
    {
        S.genes[((size_t)task * 2 + 0) * n + i] = par[i];
        S.genes[((size_t)task * 2 + 1) * n + i] = par[n + i];
        S.grads[((size_t)task * 2 + 0) * n + i] = par[2 * n + i];
        S.grads[((size_t)task * 2 + 1) * n + i] = par[3 * n + i];
    }
}

// Launch bounds = the register budget.  The 16-lane single-pose kernels run best at THREE warps per scheduler with 168 registers
// (no hot-loop spills; 16 warps per SM at 128 registers spill in the hot loop, and every other warp count from 8 to 14 was slower)
// in blocks of two warps (finer block granularity in the last wave);
// the other forms keep four warps per block and the occupancy they were tuned at.
#ifndef BIOIK_EVOLVE_WPB16
#define BIOIK_EVOLVE_WPB16 2 // warps per block of the 16-lane kernels
#endif
#ifndef BIOIK_EVOLVE_MINBLOCKS16
#define BIOIK_EVOLVE_MINBLOCKS16 6
#endif
__host__ __device__ constexpr int evolve_warps_per_block(int lpt) { return lpt == 16 ? BIOIK_EVOLVE_WPB16 : BIOIK_EVOLVE_WPB; }
#ifdef BIOIK_X_MAXNREG // experiment builds: an explicit register cap instead of a resident-block target
#define BIOIK_EVOLVE_BOUNDS(T, CH, LPT) __maxnreg__(BIOIK_X_MAXNREG)
#else
#define BIOIK_EVOLVE_BOUNDS(T, CH, LPT) __launch_bounds__(32 * evolve_warps_per_block(LPT), (LPT == 16 ? BIOIK_EVOLVE_MINBLOCKS16 : (T * CH <= 4 ? BIOIK_EVOLVE_MINBLOCKS : (T * CH <= 6 ? 3 : 2))))
#endif
template <int T, int CH, int GSPEC, bool JOINT, int NG = 0, bool TM = false, int LPT = 32> __global__ void BIOIK_EVOLVE_BOUNDS(T, CH, LPT) k_evolve_fast(const DProblem* __restrict__ Pp, DState S, int step, const double* __restrict__ mtab)
{
    extern __shared__ double smem[];
    const DProblem& P = *Pp;
    constexpr int TPW = 32 / LPT;              // tasks per warp
    const int lane = (threadIdx.x & 31) % LPT; // lane within the task's group
    const int grp = (threadIdx.x & 31) / LPT;
    const int lane0 = grp * LPT;               // first warp lane of the group
    const unsigned gmask = LPT == 32 ? 0xffffffffu : (((1u << LPT) - 1u) << lane0); // the group's lanes: every warp-level primitive of the body is group-wide
    const int warp_in_block = threadIdx.x >> 5;
    const int task = (blockIdx.x * (blockDim.x >> 5) + warp_in_block) * TPW + grp;
    const int n = NG ? NG : P.n;
    FastSmem L{n, TM ? P.T : T, P.G, JOINT ? P.n_joint_goals : 0, P.has_secondary ? 0 : 1, TM ? P.tip_gene_start[P.T] : 0};
    evolve_fast_task<T, CH, GSPEC, JOINT, NG, TM, LPT>(P, S, step, mtab, smem + (size_t)(warp_in_block * TPW + grp) * L.total(), task, lane, lane0, gmask);
}

typedef void (*EvolveFastKernel)(const DProblem*, DState, int, const double*);

// name of the kernel instantiation the last select_* call of this thread returned (bench.py's roofline.kernel)
inline const char*& selected_kernel_name()
{
    static thread_local const char* name = "";
    return name;
}
#define BIOIK_NAMED_AS(TYPE, ...) (selected_kernel_name() = #__VA_ARGS__, (TYPE)__VA_ARGS__)

// picks the instantiation for (tips, population, goals); returns nullptr if the generic kernel must be used
// *lanes_per_task (if given) receives the lane-group width of the returned kernel: the launch has 32 / width tasks per warp
inline EvolveFastKernel select_evolve_fast(const DProblem& P, int C, int ch_cap = 8, int* lanes_per_task = nullptr, int lpt_want = 16)
{
    const int T = P.T;
    if(lanes_per_task) *lanes_per_task = 32;
#ifdef BIOIK_SLIM
#ifndef BIOIK_X_CH
#define BIOIK_X_CH 4
#endif
#ifndef BIOIK_X_LPT
#define BIOIK_X_LPT 16
#endif
    if(lanes_per_task) *lanes_per_task = BIOIK_X_LPT;
    return BIOIK_NAMED_AS(EvolveFastKernel, k_evolve_fast<1, BIOIK_X_CH, 1, false, 7, false, BIOIK_X_LPT>);
#else
    if(T < 1 || T > 8 || P.n_joint_goals > FAST_MAX_JOINT_GOALS || C > 32 * FAST_MAX_CPL) return nullptr;
    if(P.n_balance > 0) return nullptr; // BalanceGoal reads every tip frame at once: the generic kernels evaluate it
    if(P.n_quat > 0) return nullptr; // quaternion genes are renormalised after the mutation (couples four genes): generic kernel
    const bool J = P.n_joint_goals > 0;
    const bool single_pose = (P.G == 1 && P.goals[0].type == G_POSE && !P.goals[0].secondary && T == 1);
    int cpl = mtab_row(C) / 32; // 1, 2, 4 or 8
    if(cpl > ch_cap) cpl = ch_cap; // experiment knob: smaller register blocks (more chunks, fewer registers)
    if(J && cpl > 2) cpl = 2;      // joint-space accumulators on top of the frame accumulators: blocks of 4 spill (cfg4 is faster with 2)
#define BIOIK_PICK(TT, CC) (J ? BIOIK_NAMED_AS(EvolveFastKernel, k_evolve_fast<TT, CC, 0, true>) : BIOIK_NAMED_AS(EvolveFastKernel, k_evolve_fast<TT, CC, 0, false>))
    if(single_pose && (P.n == 7 || P.n == 6) && ch_cap >= 8)
    {
        // lane groups: LPT lanes per task, R / (LPT * CH) chunks of CH children per lane.  R >= 128: 8, 16 or 32 lanes as wanted,
        // blocks of 4; R = 64 (population <= 66): 16 or 8 lanes; R = 32 (population <= 34, the reference's 18): 16 lanes, blocks of 2
        const int R = mtab_row(C);
        int lpt = lanes_per_task ? (lpt_want <= 8 ? 8 : (lpt_want <= 16 ? 16 : 32)) : 32;
        if(R == 64 && lpt == 32) lpt = 16;
        if(R == 32) lpt = lanes_per_task ? 16 : 32;
        if(lanes_per_task) *lanes_per_task = lpt;
#define BIOIK_PICK_LG(NN)                                                                                                                                              \
    (R == 32 ? (lpt == 16 ? BIOIK_NAMED_AS(EvolveFastKernel, k_evolve_fast<1, 2, 1, false, NN, false, 16>) : BIOIK_NAMED_AS(EvolveFastKernel, k_evolve_fast<1, 1, 1, false>))                          \
             : (lpt == 8 ? BIOIK_NAMED_AS(EvolveFastKernel, k_evolve_fast<1, 4, 1, false, NN, false, 8>) : (lpt == 16 ? BIOIK_NAMED_AS(EvolveFastKernel, k_evolve_fast<1, 4, 1, false, NN, false, 16>) : BIOIK_NAMED_AS(EvolveFastKernel, k_evolve_fast<1, 4, 1, false, NN>))))
        return P.n == 7 ? BIOIK_PICK_LG(7) : BIOIK_PICK_LG(6);
#undef BIOIK_PICK_LG
    }
    if(single_pose) return cpl >= 3 ? BIOIK_NAMED_AS(EvolveFastKernel, k_evolve_fast<1, 4, 1, false>) : (cpl == 2 ? BIOIK_NAMED_AS(EvolveFastKernel, k_evolve_fast<1, 2, 1, false>) : BIOIK_NAMED_AS(EvolveFastKernel, k_evolve_fast<1, 1, 1, false>));
    if(T == 1) return cpl >= 3 ? BIOIK_PICK(1, 4) : (cpl == 2 ? BIOIK_PICK(1, 2) : BIOIK_PICK(1, 1));
    if(!fast_tip_major(P)) return cpl >= 2 ? BIOIK_PICK(2, 2) : BIOIK_PICK(2, 1); // two tips still fit the gene-major register block (cfg3 is slightly faster that way)
    // three or more tips: the tip-major form (one tip's accumulators at a time, so the register block does not depend on T; faster on cfg5)
#define BIOIK_PICK_TM(CC) (J ? BIOIK_NAMED_AS(EvolveFastKernel, k_evolve_fast<1, CC, 0, true, 0, true>) : BIOIK_NAMED_AS(EvolveFastKernel, k_evolve_fast<1, CC, 0, false, 0, true>))
    return cpl >= 3 ? BIOIK_PICK_TM(4) : (cpl == 2 ? BIOIK_PICK_TM(2) : BIOIK_PICK_TM(1));
#undef BIOIK_PICK_TM
#undef BIOIK_PICK
#endif
}

} // namespace bioik
