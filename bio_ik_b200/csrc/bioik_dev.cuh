// bioik_dev.cuh — per-thread device functions of the H100 bio2/bio2_memetic path.
//
// Arithmetic contract (DESIGN.md §3): IEEE binary64, no implicit FMA contraction
// (nvcc -fmad=false), explicit __fma_rn only where the reference's AVX+FMA
// approximator fuses (src/forward_kinematics.h:949-950,1091-1092) and inside
// d_sincos.  Every function below states the reference lines it implements and
// keeps their operation ORDER, so results are bit-identical to an IEEE-strict
// CPU evaluation of the same formulas.
//
// The functions are written against plain pointers (global or shared memory) so
// that tests/hostsim can compile this header with g++ (BIOIK_HOSTSIM) and check
// the per-thread logic without a GPU.  That build is test-only: the shipped
// library contains CUDA kernels only.
#pragma once

#include <stdint.h>
#include <type_traits>

#ifdef BIOIK_HOSTSIM
#include <cmath>
#define BIOIK_HD inline
#define BIOIK_FMA(a, b, c) std::fma((a), (b), (c))
#define BIOIK_RINT(x) std::rint(x)
#define BIOIK_FMOD(x, y) std::fmod((x), (y))
#define BIOIK_SQRT(x) std::sqrt(x)
#define BIOIK_FABS(x) std::fabs(x)
#define BIOIK_FMIN(a, b) std::fmin((a), (b))
#define BIOIK_FMAX(a, b) std::fmax((a), (b))
#define BIOIK_FLOOR(x) std::floor(x)
#define BIOIK_CEIL(x) std::ceil(x)
#define BIOIK_ATAN2(a, b) std::atan2((a), (b))
#define BIOIK_ACOS(a) std::acos(a)
static inline double bioik_clear_low_word(double s)
{
    uint64_t b;
    __builtin_memcpy(&b, &s, 8);
    b &= 0xFFFFFFFF00000000ull;
    __builtin_memcpy(&s, &b, 8);
    return s;
}
#define BIOIK_CLEAR_LOW_WORD(s) bioik_clear_low_word(s)
static inline double bioik_sel_gt0(double c, double a, double b) { return c > 0.0 ? a : b; }
static inline double bioik_sel_ne0(double c, double a, double b) { return c != 0.0 ? a : b; }
#else
#define BIOIK_HD __device__ __forceinline__
#define BIOIK_FMA(a, b, c) __fma_rn((a), (b), (c))
#define BIOIK_RINT(x) rint(x)
#define BIOIK_FMOD(x, y) fmod((x), (y))
#define BIOIK_SQRT(x) sqrt(x)
#define BIOIK_FABS(x) fabs(x)
#define BIOIK_FMIN(a, b) fmin((a), (b))
#define BIOIK_FMAX(a, b) fmax((a), (b))
#define BIOIK_FLOOR(x) floor(x)
#define BIOIK_CEIL(x) ceil(x)
#define BIOIK_ATAN2(a, b) atan2((a), (b))
#define BIOIK_ACOS(a) acos(a)
#define BIOIK_CLEAR_LOW_WORD(s) __hiloint2double(__double2hiint(s), 0)
// c > 0 ? a : b and c != 0 ? a : b as SELECT instructions (false for a NaN c): left to itself the compiler turns such an
// expression on per-lane data into a divergent branch
__device__ __forceinline__ double bioik_sel_gt0(double c, double a, double b)
{
    double r;
    asm("{\n\t.reg .pred p;\n\tsetp.gt.f64 p, %1, 0d0000000000000000;\n\tselp.f64 %0, %2, %3, p;\n\t}" : "=d"(r) : "d"(c), "d"(a), "d"(b));
    return r;
}
__device__ __forceinline__ double bioik_sel_ne0(double c, double a, double b)
{
    double r;
    asm("{\n\t.reg .pred p;\n\tsetp.ne.f64 p, %1, 0d0000000000000000;\n\tselp.f64 %0, %2, %3, p;\n\t}" : "=d"(r) : "d"(c), "d"(a), "d"(b));
    return r;
}
#endif

namespace bioik
{

// compiled-in capacities (BIOIK_E_LIMIT beyond)
constexpr int MAX_VARS = 64;   // robot variables
constexpr int MAX_GENES = 48;  // active variables
constexpr int MAX_SLOTS = 96;  // links in the FK schedule
constexpr int MAX_TIPS = 24; // BalanceGoal makes every link with mass a tip (src/goal_types.cpp:251)
constexpr int MAX_GOALS = 24;
constexpr int GOAL_NPARAM = 12;
constexpr double DBLMAX = 1.7976931348623157e308;

enum JointType { J_FIXED = 0, J_REVOLUTE = 1, J_PRISMATIC = 2, J_FLOATING = 3, J_PLANAR = 4 };
enum GoalType {
    G_POSITION = 1, G_ORIENTATION, G_POSE, G_LOOK_AT, G_MAX_DISTANCE, G_MIN_DISTANCE, G_LINE, G_PLANE, G_AVOID_JOINT_LIMITS,
    G_CENTER_JOINTS, G_REGULARIZATION, G_MINIMAL_DISPLACEMENT, G_JOINT_VARIABLE, G_SIDE, G_DIRECTION, G_CONE, G_BALANCE
};

// ---------------------------------------------------------------------------
// Flattened problem (device constant data; built by the host in bioik_capi.cu)
// ---------------------------------------------------------------------------
struct DSlot // one scheduled link (src/forward_kinematics.h:268-282 order)
{
    int32_t parent; // schedule slot of the parent link, -1 for the root
    int32_t type;   // JointType of the parent joint
    int32_t var;    // first variable index, -1 if none
    int32_t tipmask; // bit t set: tip t depends on this joint (tip_dependencies, :588-598)
    double origin[7];
    double axis[3];
};
struct DGene // one active variable (problem.active_variables order)
{
    int32_t var;       // robot variable index
    int32_t dep_start; // range in DProblem::dep_* (joint_dependencies of the variable's joint, :570-587)
    int32_t dep_count; // 0 if the variable's own joint mimics another joint (:623)
    int32_t tipmask;   // bit t set: the variable can move tip t (OR of its dependency joints' tipmask)
    int32_t var_in_joint; // index of the variable inside its joint: the numeric Jacobian branch moves THIS variable of every dependency joint (:698-699)
    double clip_min, clip_max, span, vmin, vmax, vel_weight; // robot_info.h:48-55, problem.cpp:206-225
};
struct DGoal
{
    int32_t type, tip, secondary, var_index; // var_index: gene index or -1-robot_var (goal.h:70-77)
    double weight_sq;
};
struct DMimic
{
    int32_t dest, src;
    double factor, offset;
};
struct DProblem
{
    int32_t n_vars, n, T, L, G, n_mimic, has_secondary, n_joint_goals;
    double dpos, drot, dtwist;
    int32_t tip_slot[MAX_TIPS];
    int32_t gene_of_var[MAX_VARS]; // -1 if inactive
    DSlot slots[MAX_SLOTS];
    DGene genes[MAX_GENES];
    DGoal goals[MAX_GOALS];
    DMimic mimics[MAX_VARS];
    int32_t dep_slot[MAX_SLOTS + MAX_GENES];
    double dep_scale[MAX_SLOTS + MAX_GENES];
    int32_t tip_gene_start[MAX_TIPS + 1]; // genes that can move tip t (DGene::tipmask), ascending: tip_gene[tip_gene_start[t] .. tip_gene_start[t + 1])
    int16_t tip_gene[MAX_TIPS * MAX_GENES];
    int32_t n_quat;               // floating joints among the genes: quat_gene[k] = gene of rot_x, the next three genes are rot_y, rot_z, rot_w (ik_evolution_2.cpp:118-126)
    int32_t quat_gene[MAX_GENES / 4];
    int32_t wrap_gene[MAX_GENES]; // 1: the plugin's angle wrap applies (revolute variable, robot without mimic joints; kinematics_plugin.cpp:583-584)
    // BalanceGoal::balance_infos (src/goal_types.cpp:236-259): the links with mass in link order - their tip index, inertial origin
    // and mass / total mass
    int32_t n_balance;
    int32_t balance_tip[MAX_TIPS];
    double balance_center[MAX_TIPS][3];
    double balance_weight[MAX_TIPS];
};

// ---------------------------------------------------------------------------
// frames as 7 doubles: px py pz qx qy qz qw   (include/bio_ik/frame.h)
// ---------------------------------------------------------------------------
struct V3 { double x, y, z; };
struct Q4 { double x, y, z, w; };
struct F7 { V3 p; Q4 q; };

// Strided view: element e lives at p[e * s].  The fused serial kernel keeps per-thread arrays as
// shared-memory COLUMNS (s = blockDim.x) so that a warp's accesses are bank-conflict free; plain
// pointers (s = 1) work with the same templated functions.
template <class E> struct ColT
{
    E* p;
    int s;
    BIOIK_HD E& operator[](int e) const { return p[(size_t)e * s]; }
    BIOIK_HD ColT operator+(int e) const { return ColT{p + (size_t)e * s, s}; }
    template <class U = E, class = typename std::enable_if<!std::is_const<U>::value>::type> BIOIK_HD operator ColT<const E>() const { return ColT<const E>{p, s}; }
    BIOIK_HD explicit operator bool() const { return p != nullptr; }
};
typedef ColT<double> Col;
typedef ColT<const double> CCol;

// same with a compile-time stride (lets the compiler fold the stride into immediates and keep the
// shared-memory address space of the base pointer)
template <class E, int S> struct FixedCol
{
    E* p;
    BIOIK_HD E& operator[](int e) const { return p[e * S]; }
    BIOIK_HD FixedCol operator+(int e) const { return FixedCol{p + e * S}; }
    template <class U = E, class = typename std::enable_if<!std::is_const<U>::value>::type> BIOIK_HD operator FixedCol<const E, S>() const { return FixedCol<const E, S>{p}; }
};

template <class A> BIOIK_HD F7 load_frame(A f) { return F7{{f[0], f[1], f[2]}, {f[3], f[4], f[5], f[6]}}; }
template <class A> BIOIK_HD void store_frame(A f, const F7& a)
{
    f[0] = a.p.x; f[1] = a.p.y; f[2] = a.p.z; f[3] = a.q.x; f[4] = a.q.y; f[5] = a.q.z; f[6] = a.q.w;
}

// include/bio_ik/frame.h:108-149.  The early-out (:122-126) returns exactly what the
// arithmetic below produces for those inputs (up to the sign of zero), so it is dropped.
BIOIK_HD V3 quat_mul_vec(const Q4& q, const V3& v)
{
    double t_x = q.y * v.z - q.z * v.y;
    double t_y = q.z * v.x - q.x * v.z;
    double t_z = q.x * v.y - q.y * v.x;
    double r_x = q.w * t_x + q.y * t_z - q.z * t_y;
    double r_y = q.w * t_y + q.z * t_x - q.x * t_z;
    double r_z = q.w * t_z + q.x * t_y - q.y * t_x;
    r_x += r_x; r_y += r_y; r_z += r_z;
    r_x += v.x; r_y += v.y; r_z += v.z;
    return V3{r_x, r_y, r_z};
}
// include/bio_ik/frame.h:151-172
BIOIK_HD Q4 quat_mul_quat(const Q4& p, const Q4& q)
{
    Q4 r;
    r.x = (p.w * q.x + p.x * q.w) + (p.y * q.z - p.z * q.y);
    r.y = (p.w * q.y - p.x * q.z) + (p.y * q.w + p.z * q.x);
    r.z = (p.w * q.z + p.x * q.y) - (p.y * q.x - p.z * q.w);
    r.w = (p.w * q.w - p.x * q.x) - (p.y * q.y + p.z * q.z);
    return r;
}
// tf2::operator*(Quaternion, Quaternion), left-to-right (used by computeJacobian :648,:680)
BIOIK_HD Q4 tf2_mul(const Q4& a, const Q4& b)
{
    Q4 r;
    r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
    r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
    r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
    r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
    return r;
}
BIOIK_HD Q4 quat_inv(const Q4& q) { return Q4{-q.x, -q.y, -q.z, q.w}; }
// include/bio_ik/frame.h:174-180
BIOIK_HD F7 concat(const F7& a, const F7& b)
{
    V3 d = quat_mul_vec(a.q, b.p);
    F7 r;
    r.p = V3{a.p.x + d.x, a.p.y + d.y, a.p.z + d.z};
    r.q = quat_mul_quat(a.q, b.q);
    return r;
}

// The quat_mul_vec early-out matters in ONE way: when v == 0 or q == identity the
// reference returns v itself.  The arithmetic path returns the same VALUE; only a
// negative zero could differ, and no later operation distinguishes signed zeros.

// d_sincos: arithmetic-contract sin/cos (DESIGN.md §3) of the half joint angle
// (src/forward_kinematics.h:99-104): Cody–Waite reduction by pi/2 with explicit FMA,
// fdlibm minimax polynomials; identical operation sequence on CPU oracle and GPU.
BIOIK_HD void d_sincos(double x, double& s_out, double& c_out)
{
    if(!(BIOIK_FABS(x) <= 1.0e5)) x = BIOIK_FMOD(x, 6.283185307179586);
    double fn = BIOIK_RINT(x * 0.6366197723675814);
    double r = BIOIK_FMA(fn, -1.5707963267948966, x);
    r = BIOIK_FMA(fn, -6.123233995736766e-17, r);
    r = BIOIK_FMA(fn, 1.4973849048591698e-33, r);
    double z = r * r;
    double ps = BIOIK_FMA(z, 1.58969099521155010221e-10, -2.50507602534068634195e-08);
    ps = BIOIK_FMA(z, ps, 2.75573137070700676789e-06);
    ps = BIOIK_FMA(z, ps, -1.98412698298579493134e-04);
    ps = BIOIK_FMA(z, ps, 8.33333333332248946124e-03);
    ps = BIOIK_FMA(z, ps, -1.66666666666666324348e-01);
    double sr = BIOIK_FMA(r * z, ps, r);
    double pc = BIOIK_FMA(z, -1.13596475577881948265e-11, 2.08757232129817482790e-09);
    pc = BIOIK_FMA(z, pc, -2.75573143513906633035e-07);
    pc = BIOIK_FMA(z, pc, 2.48015872894767294178e-05);
    pc = BIOIK_FMA(z, pc, -1.38888888888741095749e-03);
    pc = BIOIK_FMA(z, pc, 4.16666666666666019037e-02);
    double cr = BIOIK_FMA(z * z, pc, BIOIK_FMA(z, -0.5, 1.0));
    long long q = (long long)fn;
    double s = (q & 1) ? cr : sr;
    double c = (q & 1) ? sr : cr;
    if(q & 2) s = -s;
    if((q + 1) & 2) c = -c;
    s_out = s;
    c_out = c;
}

// d_acos: arithmetic-contract acos of ConeGoal (fdlibm e_acos.c algorithm, IEEE operations only): identical
// operation sequence in the CPU oracle (det_acos).
BIOIK_HD double d_acos(double x)
{
    const double one = 1.0, pi = 3.14159265358979311600e+00, pio2_hi = 1.57079632679489655800e+00, pio2_lo = 6.12323399573676603587e-17;
    const double pS0 = 1.66666666666666657415e-01, pS1 = -3.25565818622400915405e-01, pS2 = 2.01212532134862925881e-01, pS3 = -4.00555345006794114027e-02, pS4 = 7.91534994289814532176e-04,
                 pS5 = 3.47933107596021167570e-05;
    const double qS1 = -2.40339491173441421878e+00, qS2 = 2.02094576023350569471e+00, qS3 = -6.88283971605453293030e-01, qS4 = 7.70381505559019352791e-02;
    const double ax = BIOIK_FABS(x);
    if(!(ax < 1.0))
    {
        if(x == 1.0) return 0.0;
        if(x == -1.0) return pi + 2.0 * pio2_lo;
        return (x - x) / (x - x);
    }
    if(ax < 0.5)
    {
        if(ax < 6.938893903907228e-18) return pio2_hi + pio2_lo;
        double z = x * x;
        double p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
        double q = one + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
        double r = p / q;
        return pio2_hi - (x - (pio2_lo - x * r));
    }
    if(x < 0)
    {
        double z = (one + x) * 0.5;
        double p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
        double q = one + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
        double s = BIOIK_SQRT(z);
        double r = p / q;
        double w = r * s - pio2_lo;
        return pi - 2.0 * (s + w);
    }
    double z = (one - x) * 0.5;
    double s = BIOIK_SQRT(z);
    double df = BIOIK_CLEAR_LOW_WORD(s);
    double c = (z - df * df) / (s + df);
    double p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
    double q = one + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
    double r = p / q;
    double w = r * s + c;
    return 2.0 * (df + w);
}

// goal_types.h:700-711 on a frame f (px py pz qx qy qz qw)
template <class AP, class AF> BIOIK_HD double cone_goal_value(AP p, AF f)
{
    double sum = 0.0;
    V3 v = quat_mul_vec(Q4{f[3], f[4], f[5], f[6]}, V3{p[4], p[5], p[6]});
    double s = BIOIK_SQRT((v.x * v.x + v.y * v.y + v.z * v.z) * (p[7] * p[7] + p[8] * p[8] + p[9] * p[9]));
    double c = (v.x * p[7] + v.y * p[8] + v.z * p[9]) / s;
    if(c < -1.0) c = -1.0;
    if(c > 1.0) c = 1.0;
    double d = BIOIK_FMAX(0.0, d_acos(c) - p[10]);
    sum += d * d;
    double w = p[3];
    double dx = p[0] - f[0], dy = p[1] - f[1], dz = p[2] - f[2];
    sum += w * w * (dx * dx + dy * dy + dz * dz);
    return sum;
}

// src/utils.h:319
BIOIK_HD double mix(double a, double b, double f) { return a * (1.0 - f) + b * f; }
// src/utils.h:321-326 / robot_info.h:61-66 (NaN passes through, like the reference)
BIOIK_HD double clampd(double v, double lo, double hi)
{
    if(v < lo) v = lo;
    if(v > hi) v = hi;
    return v;
}

// ---------------------------------------------------------------------------
// variable vector of a task: seed with the active entries replaced by genes
// (genesToJointVariables, src/ik_evolution_2.cpp:101-107) then updateMimic
// (src/forward_kinematics.h:230-246)
// ---------------------------------------------------------------------------
template <class AS, class AG, class AV> BIOIK_HD void assemble_variables(const DProblem& P, AS seed, AG genes, AV vars)
{
    for(int v = 0; v < P.n_vars; v++)
    {
        int g = P.gene_of_var[v];
        vars[v] = g >= 0 ? genes[g] : seed[v];
    }
    for(int m = 0; m < P.n_mimic; m++) vars[P.mimics[m].dest] = vars[P.mimics[m].src] * P.mimics[m].factor + P.mimics[m].offset;
}

// PLANAR joint (:128-135): MoveIt's computeTransform = Translation3d(x, y, 0) * AngleAxisd(theta, UnitZ()), Eigen's
// AngleAxis::toRotationMatrix for that axis = [[c, -s, 0], [s, c, 0], [0, 0, (1 - c) + c]], then Frame(Isometry3d)
// (include/bio_ik/frame.h:74-79) with Eigen's matrix -> quaternion (Shoemake).  Third-party arithmetic restated.
BIOIK_HD F7 planar_frame(double x, double y, double theta)
{
    double s, c;
    d_sincos(theta, s, c);
    const double m00 = 0.0 * 0.0 + c, m01 = 0.0 - s, m10 = 0.0 + s, m11 = 0.0 * 0.0 + c, m22 = (1.0 - c) * 1.0 + c;
    F7 f;
    f.p = V3{x, y, 0.0};
    double t = m00 + m11 + m22;
    if(t > 0.0)
    {
        t = BIOIK_SQRT(t + 1.0);
        const double w = 0.5 * t;
        t = 0.5 / t;
        f.q = Q4{(0.0 - 0.0) * t, (0.0 - 0.0) * t, (m10 - m01) * t, w};
    }
    else if(m22 > m00)
    {
        t = BIOIK_SQRT(m22 - m00 - m11 + 1.0);
        const double z = 0.5 * t;
        t = 0.5 / t;
        f.q = Q4{(0.0 + 0.0) * t, (0.0 + 0.0) * t, z, (m10 - m01) * t};
    }
    else
    {
        t = BIOIK_SQRT(m00 - m11 - m22 + 1.0);
        const double xx = 0.5 * t;
        t = 0.5 / t;
        f.q = Q4{xx, (m10 + m01) * t, (0.0 + 0.0) * t, (0.0 - 0.0) * t};
    }
    return f;
}

// joint-local frame, src/forward_kinematics.h:78-139
template <class AV> BIOIK_HD F7 joint_frame(const DSlot& S, AV vars)
{
    F7 f;
    f.p = V3{0.0, 0.0, 0.0};
    f.q = Q4{0.0, 0.0, 0.0, 1.0};
    if(S.type == J_REVOLUTE)
    {
        double half_angle = vars[S.var] * 0.5;
        double fs, fc;
        d_sincos(half_angle, fs, fc);
        f.q = Q4{S.axis[0] * fs, S.axis[1] * fs, S.axis[2] * fs, fc};
    }
    else if(S.type == J_PRISMATIC)
    {
        double v = vars[S.var];
        f.p = V3{S.axis[0] * v, S.axis[1] * v, S.axis[2] * v};
    }
    else if(S.type == J_FLOATING) // :120-127: translation + normalised quaternion (tf2 normalized(): q * (1 / length))
    {
        f.p = V3{vars[S.var + 0], vars[S.var + 1], vars[S.var + 2]};
        const double x = vars[S.var + 3], y = vars[S.var + 4], z = vars[S.var + 5], w = vars[S.var + 6];
        const double sc = 1.0 / BIOIK_SQRT(x * x + y * y + z * z + w * w);
        f.q = Q4{x * sc, y * sc, z * sc, w * sc};
    }
    else if(S.type == J_PLANAR)
        f = planar_frame(vars[S.var + 0], vars[S.var + 1], vars[S.var + 2]);
    return f;
}
// the same with variable `which` of the joint moved by `dv` (numeric differentiation, :700-704)
template <class AV> BIOIK_HD F7 joint_frame_moved(const DSlot& S, AV vars, int which, double dv)
{
    double v[7];
    const int cnt = S.type == J_PLANAR ? 3 : 7;
    for(int k = 0; k < cnt; k++) v[k] = vars[S.var + k];
    if(which < cnt) v[which] = v[which] + dv; // a joint that mimics a joint with more variables: variables[ivar2] lies outside it, its frame does not move
    if(S.type == J_PLANAR) return planar_frame(v[0], v[1], v[2]);
    F7 f;
    f.p = V3{v[0], v[1], v[2]};
    const double sc = 1.0 / BIOIK_SQRT(v[3] * v[3] + v[4] * v[4] + v[5] * v[5] + v[6] * v[6]);
    f.q = Q4{v[3] * sc, v[4] * sc, v[5] * sc, v[6] * sc};
    return f;
}

// include/bio_ik/frame.h:189-209
BIOIK_HD F7 frame_invert(const F7& a)
{
    F7 r;
    r.q = quat_inv(a.q);
    r.p = quat_mul_vec(r.q, V3{-a.p.x, -a.p.y, -a.p.z});
    return r;
}
// change(a, b, c) = a * inverse(b) * c, bracketed like concat(a, tmp, c, r)
BIOIK_HD F7 frame_change(const F7& a, const F7& b, const F7& c) { return concat(concat(a, frame_invert(b)), c); }

// RobotFK_Fast_Base::applyConfiguration, src/forward_kinematics.h:331-354.
// frames: [L][7] scratch (global frames of the scheduled links).
template <class AV, class AF> BIOIK_HD void exact_fk(const DProblem& P, AV vars, AF frames)
{
    for(int s = 0; s < P.L; s++)
    {
        const DSlot& S = P.slots[s];
        F7 jf = joint_frame(S, vars);
        F7 o = load_frame(S.origin);
        F7 r;
        if(S.parent >= 0)
            r = concat(concat(load_frame(frames + 7 * S.parent), o), jf);
        else
            r = concat(o, jf);
        store_frame(frames + 7 * s, r);
    }
}

// RobotFK_Jacobian::computeJacobian (src/forward_kinematics.h:600-730) fused with
// RobotFK_Mutator::initializeMutationApproximator (:802-930) for one (gene, tip):
// returns the delta frame; *masked = the :919-926 test.
// vars: the post-mimic variables the frames were computed from (read only by the numeric branch of floating joints)
template <class AF, class AV> BIOIK_HD F7 delta_frame(const DProblem& P, AF frames, AV vars, int gene, int tip, bool& masked)
{
    const DGene& Gn = P.genes[gene];
    F7 tipf = load_frame(frames + 7 * P.tip_slot[tip]);
    double j0 = 0, j1 = 0, j2 = 0, j3 = 0, j4 = 0, j5 = 0;
    for(int d = 0; d < Gn.dep_count; d++)
    {
        int s = P.dep_slot[Gn.dep_start + d];
        double scale = P.dep_scale[Gn.dep_start + d];
        const DSlot& S = P.slots[s];
        if(!((S.tipmask >> tip) & 1)) continue;
        F7 lf = load_frame(frames + 7 * s);
        if(S.type == J_REVOLUTE)
        {
            Q4 q = tf2_mul(quat_inv(lf.q), tipf.q); // :648
            q = quat_inv(q);                        // :649
            V3 rot = quat_mul_vec(q, V3{S.axis[0], S.axis[1], S.axis[2]}); // :651-652
            V3 vel = V3{lf.p.x - tipf.p.x, lf.p.y - tipf.p.y, lf.p.z - tipf.p.z}; // :654
            vel = quat_mul_vec(quat_inv(tipf.q), vel);                            // :655
            V3 c = V3{vel.y * rot.z - vel.z * rot.y, vel.z * rot.x - vel.x * rot.z, vel.x * rot.y - vel.y * rot.x}; // :657
            j0 += c.x * scale; j1 += c.y * scale; j2 += c.z * scale;
            j3 += rot.x * scale; j4 += rot.y * scale; j5 += rot.z * scale;
        }
        else if(S.type == J_PRISMATIC)
        {
            Q4 q = tf2_mul(quat_inv(lf.q), tipf.q); // :680
            q = quat_inv(q);
            V3 v = quat_mul_vec(q, V3{S.axis[0], S.axis[1], S.axis[2]}); // :685
            j0 += v.x * scale; j1 += v.y * scale; j2 += v.z * scale;
        }
        else if(S.type == J_FLOATING || S.type == J_PLANAR)
        {
            // numeric differentiation (:695-726): move this variable by 1e-5, rebuild the link frame, carry the tip along
            // (change) and take the twist between the two tip frames (frameTwist, include/bio_ik/frame.h:240-259)
            const double step_size = 0.00001, inv_step_size = 1.0 / step_size;
            // ivar2 (:698-699): the variable itself for its own joint, the same position inside a joint that mimics it
            const F7 jf2 = joint_frame_moved(S, vars, Gn.var_in_joint, step_size);
            const F7 o = load_frame(S.origin);
            const F7 link2 = S.parent >= 0 ? concat(concat(load_frame(frames + 7 * S.parent), o), jf2) : concat(o, jf2);
            const F7 tip2 = frame_change(link2, lf, tipf);
            const F7 rel = concat(frame_invert(tipf), tip2); // inverse(a) * b
            double w = rel.q.w; // Quaternion::getAngle = 2 acos(w), tf2Acos clamps
            if(w < -1.0) w = -1.0;
            if(w > 1.0) w = 1.0;
            double ra = 2.0 * d_acos(w);
            if(ra > 3.14159265358979323846) ra -= 2 * 3.14159265358979323846;
            const double s_squared = 1.0 - rel.q.w * rel.q.w; // Quaternion::getAxis
            V3 ax = V3{1.0, 0.0, 0.0};
            if(!(s_squared < 10.0 * 2.2204460492503131e-16))
            {
                const double sq = BIOIK_SQRT(s_squared);
                ax = V3{rel.q.x / sq, rel.q.y / sq, rel.q.z / sq};
            }
            j0 += rel.p.x * inv_step_size * scale; j1 += rel.p.y * inv_step_size * scale; j2 += rel.p.z * inv_step_size * scale;
            j3 += ax.x * ra * inv_step_size * scale; j4 += ax.y * ra * inv_step_size * scale; j5 += ax.z * ra * inv_step_size * scale;
        }
    }
    F7 d;
    d.p = quat_mul_vec(tipf.q, V3{j0, j1, j2}); // :833-838
    Q4 q = quat_mul_quat(tipf.q, Q4{j3 * 0.5, j4 * 0.5, j5 * 0.5, 1.0}); // :842-847
    d.q = Q4{q.x - tipf.q.x, q.y - tipf.q.y, q.z - tipf.q.z, q.w - tipf.q.w}; // :848
    masked = (d.p.x != 0.0) | (d.p.y != 0.0) | (d.p.z != 0.0) | (d.q.x != 0.0) | (d.q.y != 0.0) | (d.q.z != 0.0); // :919-926
    // A gene outside mutation_approx_map contributes nothing (:1083,:1198); a zero delta frame
    // makes the dense loops below add exactly 0.
    if(!masked) d.q.w = 0.0;
    return d;
}

// computeApproximateMutations for one genotype, src/forward_kinematics.h:1061-1110 (AVX+FMA form).
// tip0 [T][7], delta [T][n][7] (zero where unmasked), base [n], x [n] -> out [T][7]
// Same, skipping (tip, gene) pairs that are structurally independent (DGene::tipmask): their delta frame is
// all-zero, and fma(d, 0, f) == f, so the result is unchanged.
template <class A0, class AD, class AB, class AX, class AO> BIOIK_HD void approx_frames_sparse(const DProblem& P, A0 tip0, AD delta, AB base, AX x, AO out)
{
    const int T = P.T, n = P.n;
    for(int t = 0; t < T; t++)
    {
        double f0 = tip0[7 * t + 0], f1 = tip0[7 * t + 1], f2 = tip0[7 * t + 2], f3 = tip0[7 * t + 3], f4 = tip0[7 * t + 4], f5 = tip0[7 * t + 5], f6 = tip0[7 * t + 6];
        AD D = delta + t * n * 7;
        for(int i = 0; i < n; i++)
        {
            if(!((P.genes[i].tipmask >> t) & 1)) continue;
            double d = x[i] - base[i]; // :1086
            f0 = BIOIK_FMA(d, D[7 * i + 0], f0);
            f1 = BIOIK_FMA(d, D[7 * i + 1], f1);
            f2 = BIOIK_FMA(d, D[7 * i + 2], f2);
            f3 = BIOIK_FMA(d, D[7 * i + 3], f3);
            f4 = BIOIK_FMA(d, D[7 * i + 4], f4);
            f5 = BIOIK_FMA(d, D[7 * i + 5], f5);
            f6 = BIOIK_FMA(d, D[7 * i + 6], f6);
        }
        out[7 * t + 0] = f0; out[7 * t + 1] = f1; out[7 * t + 2] = f2; out[7 * t + 3] = f3; out[7 * t + 4] = f4; out[7 * t + 5] = f5; out[7 * t + 6] = f6;
    }
}

template <class A0, class AD, class AB, class AX, class AO> BIOIK_HD void approx_frames(int T, int n, A0 tip0, AD delta, AB base, AX x, AO out)
{
    for(int t = 0; t < T; t++)
    {
        double f0 = tip0[7 * t + 0], f1 = tip0[7 * t + 1], f2 = tip0[7 * t + 2], f3 = tip0[7 * t + 3], f4 = tip0[7 * t + 4], f5 = tip0[7 * t + 5], f6 = tip0[7 * t + 6];
        AD D = delta + t * n * 7;
        for(int i = 0; i < n; i++)
        {
            double d = x[i] - base[i]; // :1086
            f0 = BIOIK_FMA(d, D[7 * i + 0], f0);
            f1 = BIOIK_FMA(d, D[7 * i + 1], f1);
            f2 = BIOIK_FMA(d, D[7 * i + 2], f2);
            f3 = BIOIK_FMA(d, D[7 * i + 3], f3);
            f4 = BIOIK_FMA(d, D[7 * i + 4], f4);
            f5 = BIOIK_FMA(d, D[7 * i + 5], f5);
            f6 = BIOIK_FMA(d, D[7 * i + 6], f6);
        }
        out[7 * t + 0] = f0; out[7 * t + 1] = f1; out[7 * t + 2] = f2; out[7 * t + 3] = f3; out[7 * t + 4] = f4; out[7 * t + 5] = f5; out[7 * t + 6] = f6;
    }
}

// computeApproximateMutation1, src/forward_kinematics.h:933-964 (AVX+FMA form), with the
// intended semantics for tips the variable does not influence (zero delta => copy; SURVEY.md Q2)
template <class AD, class AI, class AO> BIOIK_HD void approx_frames1(int T, int n, AD delta, int gene, double dv, AI in, AO out)
{
    for(int t = 0; t < T; t++)
    {
        AD D = delta + (t * n + gene) * 7;
        for(int k = 0; k < 7; k++) out[7 * t + k] = BIOIK_FMA(dv, D[k], in[7 * t + k]);
    }
}

// ---------------------------------------------------------------------------
// Goal::evaluate bodies (include/bio_ik/goal_types.h) * weight_sq, summed in goal
// order (src/problem.cpp:244-257).  tips [T][7], x [n] genes, gp [G][NPARAM] per-query
// goal parameters, seed [n_vars] = Problem::initial_guess.
// which: 0 = primary goals, 1 = secondary goals.
// ---------------------------------------------------------------------------
BIOIK_HD double len2(double x, double y, double z) { return x * x + y * y + z * z; }
BIOIK_HD double qlen2(double x, double y, double z, double w) { return x * x + y * y + z * z + w * w; }

template <class AP, class AT, class AX, class AS> BIOIK_HD double goal_value(const DProblem& P, const DGoal& g, AP p, AT tips, AX x, AS seed)
{
    AT f = tips + 7 * g.tip;
    switch(g.type)
    {
    case G_POSITION: // goal_types.h:96: tf2 distance2(v) = (v - this).length2()
        return len2(p[0] - f[0], p[1] - f[1], p[2] - f[2]);
    case G_ORIENTATION: // goal_types.h:119
        return BIOIK_FMIN(qlen2(p[3] - f[3], p[4] - f[4], p[5] - f[5], p[6] - f[6]), qlen2(p[3] + f[3], p[4] + f[4], p[5] + f[5], p[6] + f[6]));
    case G_POSE: // goal_types.h:149-180
    {
        double e = 0.0;
        e += len2(p[0] - f[0], p[1] - f[1], p[2] - f[2]);
        e += BIOIK_FMIN(qlen2(p[3] - f[3], p[4] - f[4], p[5] - f[5], p[6] - f[6]), qlen2(p[3] + f[3], p[4] + f[4], p[5] + f[5], p[6] + f[6])) * (p[7] * p[7]);
        return e;
    }
    case G_LOOK_AT: // goal_types.h:204-211
    {
        V3 axis = quat_mul_vec(Q4{f[3], f[4], f[5], f[6]}, V3{p[0], p[1], p[2]});
        double ax = p[3] - f[0], ay = p[4] - f[1], az = p[5] - f[2];
        double sa = 1.0 / BIOIK_SQRT(len2(ax, ay, az));
        ax = ax * sa; ay = ay * sa; az = az * sa;
        double sb = 1.0 / BIOIK_SQRT(len2(axis.x, axis.y, axis.z));
        double bx = axis.x * sb, by = axis.y * sb, bz = axis.z * sb;
        return len2(bx - ax, by - ay, bz - az);
    }
    case G_MAX_DISTANCE: // goal_types.h:235-240
    {
        double d = BIOIK_FMAX(0.0, BIOIK_SQRT(len2(p[0] - f[0], p[1] - f[1], p[2] - f[2])) - p[3]);
        return d * d;
    }
    case G_MIN_DISTANCE: // goal_types.h:264-269
    {
        double d = BIOIK_FMAX(0.0, p[3] - BIOIK_SQRT(len2(p[0] - f[0], p[1] - f[1], p[2] - f[2])));
        return d * d;
    }
    case G_LINE: // goal_types.h:293-297
    {
        double rx = f[0] - p[0], ry = f[1] - p[1], rz = f[2] - p[2];
        double k = p[3] * rx + p[4] * ry + p[5] * rz; // direction.dot(fb.pos - position)
        double qx = f[0] - p[3] * k, qy = f[1] - p[4] * k, qz = f[2] - p[5] * k;
        return len2(qx - p[0], qy - p[1], qz - p[2]);
    }
    case G_PLANE: // goal_types.h:321-327
    {
        double sd = (f[0] - p[0]) * p[3] + (f[1] - p[1]) * p[4] + (f[2] - p[2]) * p[5];
        return sd * sd;
    }
    case G_AVOID_JOINT_LIMITS: // goal_types.h:387-401
    {
        double sum = 0.0;
        for(int i = 0; i < P.n; i++)
        {
            const DGene& Gn = P.genes[i];
            if(Gn.clip_max == DBLMAX) continue;
            double d = x[i] - (Gn.vmin + Gn.vmax) * 0.5;
            d = BIOIK_FMAX(0.0, BIOIK_FABS(d) * 2.0 - Gn.span * 0.5);
            d *= Gn.vel_weight;
            sum += d * d;
        }
        return sum;
    }
    case G_CENTER_JOINTS: // goal_types.h:412-425
    {
        double sum = 0.0;
        for(int i = 0; i < P.n; i++)
        {
            const DGene& Gn = P.genes[i];
            if(Gn.clip_max == DBLMAX) continue;
            double d = x[i] - (Gn.vmin + Gn.vmax) * 0.5;
            d *= Gn.vel_weight;
            sum += d * d;
        }
        return sum;
    }
    case G_REGULARIZATION: // goal_types.h:435-444
    {
        double sum = 0.0;
        for(int i = 0; i < P.n; i++)
        {
            double d = x[i] - seed[P.genes[i].var];
            sum += d * d;
        }
        return sum;
    }
    case G_MINIMAL_DISPLACEMENT: // goal_types.h:455-465
    {
        double sum = 0.0;
        for(int i = 0; i < P.n; i++)
        {
            double d = x[i] - seed[P.genes[i].var];
            d *= P.genes[i].vel_weight;
            sum += d * d;
        }
        return sum;
    }
    case G_JOINT_VARIABLE: // goal_types.h:494-498
    {
        double v = g.var_index >= 0 ? x[g.var_index] : seed[-1 - g.var_index];
        double d = p[0] - v;
        return d * d;
    }
    case G_SIDE: // goal_types.h:606-613
    {
        V3 v = quat_mul_vec(Q4{f[3], f[4], f[5], f[6]}, V3{p[0], p[1], p[2]});
        double s = BIOIK_FMAX(0.0, v.x * p[3] + v.y * p[4] + v.z * p[5]);
        return s * s;
    }
    case G_DIRECTION: // goal_types.h:637-643
    {
        V3 v = quat_mul_vec(Q4{f[3], f[4], f[5], f[6]}, V3{p[0], p[1], p[2]});
        return len2(p[3] - v.x, p[4] - v.y, p[5] - v.z);
    }
    case G_CONE: return cone_goal_value(p, f);
    case G_BALANCE: // src/goal_types.cpp:261-272 (tf2 operator order: c * w component-wise, then +=; dot = x x' + y y' + z z')
    {
        double cx = 0.0, cy = 0.0, cz = 0.0;
        for(int i = 0; i < P.n_balance; i++)
        {
            AT fr = tips + 7 * P.balance_tip[i];
            V3 c = quat_mul_vec(Q4{fr[3], fr[4], fr[5], fr[6]}, V3{P.balance_center[i][0], P.balance_center[i][1], P.balance_center[i][2]});
            c.x += fr[0]; c.y += fr[1]; c.z += fr[2];
            const double w = P.balance_weight[i];
            cx += c.x * w; cy += c.y * w; cz += c.z * w;
        }
        cx -= p[0]; cy -= p[1]; cz -= p[2];
        const double k = p[3] * cx + p[4] * cy + p[5] * cz; // axis_.dot(center)
        cx -= p[3] * k; cy -= p[4] * k; cz -= p[5] * k;
        return len2(cx, cy, cz);
    }
    default: return 0.0;
    }
}

// IKBase::null_tip_frames (src/ik_base.h:135,160,163): what secondary goals receive instead of
// tip frames.  Uninitialised memory in the reference; identity frames here and in the oracle.
// (an identity frame per tip)
#define BIOIK_ID7 0, 0, 0, 0, 0, 0, 1
#define BIOIK_ID7x8 BIOIK_ID7, BIOIK_ID7, BIOIK_ID7, BIOIK_ID7, BIOIK_ID7, BIOIK_ID7, BIOIK_ID7, BIOIK_ID7
#ifdef BIOIK_HOSTSIM
static const double NULL_TIPS[MAX_TIPS * 7] = {BIOIK_ID7x8, BIOIK_ID7x8, BIOIK_ID7x8};
#else
static __device__ const double NULL_TIPS[MAX_TIPS * 7] = {BIOIK_ID7x8, BIOIK_ID7x8, BIOIK_ID7x8};
#endif
static_assert(MAX_TIPS == 24, "NULL_TIPS lists 24 identity frames");

template <class AP, class AT, class AX, class AS> BIOIK_HD double goal_fitness_t(const DProblem& P, int which, AP gp, AT tips, AX x, AS seed)
{
    double sum = 0.0;
    for(int g = 0; g < P.G; g++)
    {
        if(P.goals[g].secondary != which) continue;
        sum += goal_value(P, P.goals[g], gp + g * GOAL_NPARAM, tips, x, seed) * P.goals[g].weight_sq;
    }
    return sum;
}
// secondary goals (which = 1) evaluated on the null tip frames
template <class AP, class AX, class AS> BIOIK_HD double goal_fitness_secondary(const DProblem& P, AP gp, AX x, AS seed)
{
    const double* nt = NULL_TIPS;
    return goal_fitness_t(P, 1, gp, nt, x, seed);
}

BIOIK_HD double goal_fitness(const DProblem& P, int which, const double* gp, const double* tips, const double* x, const double* seed)
{
    if(!tips) tips = NULL_TIPS;
    double sum = 0.0;
    for(int g = 0; g < P.G; g++)
    {
        if(P.goals[g].secondary != which) continue;
        sum += goal_value(P, P.goals[g], gp + g * GOAL_NPARAM, tips, x, seed) * P.goals[g].weight_sq;
    }
    return sum;
}

// ---------------------------------------------------------------------------
// What the MoveIt plugin does with the solver's answer (src/kinematics_plugin.cpp:580-611): revolute variables are
// moved by multiples of 2 pi next to the initial guess, wrapped back inside their limits and clamped.
// v = solution value, r = initial guess, [lo, hi] = RobotInfo::getMin/getMax.
// ---------------------------------------------------------------------------
BIOIK_HD double wrap_angle(double v, double r, double lo, double hi)
{
    const double pi = 3.14159265358979323846;
    if(r < v - pi || r > v + pi) // move close to initial guess (:590-598)
    {
        v -= r;
        v /= (2 * pi);
        v += 0.5;
        v -= BIOIK_FLOOR(v);
        v -= 0.5;
        v *= (2 * pi);
        v += r;
    }
    if(v > hi) v -= BIOIK_CEIL(BIOIK_FMAX(0.0, v - hi) / (2 * pi)) * (2 * pi); // wrap at joint limits (:601-604)
    if(v < lo) v += BIOIK_CEIL(BIOIK_FMAX(0.0, lo - v) / (2 * pi)) * (2 * pi);
    if(v < lo) v = lo; // clamp at edges (:607-610)
    if(v > hi) v = hi;
    return v;
}

// IKParallel::solve's choice among its solver threads (src/ik_parallel.h:218-258), here among the `islands`
// differently seeded runs of one query: the successful island with the smallest primary (+ secondary, if the problem
// has secondary goals) fitness; if none succeeded, the smallest primary fitness.  Strict '<' scans in island order.
// sol: [islands][n_vars] full variable vectors, fit / succ: [islands].  Returns the island; *best = best_fitness.
template <class AP> BIOIK_HD int select_island(const DProblem& P, int islands, AP gp, const double* seed, const double* sol, const double* fit, const int32_t* succ, double* best)
{
    int best_index = 0;
    double best_fitness = DBLMAX;
    for(int i = 0; i < islands; i++)
    {
        if(!succ[i]) continue;
        double fitness = fit[i];
        if(P.has_secondary)
        {
            double x[MAX_GENES];
            for(int g = 0; g < P.n; g++) x[g] = sol[(size_t)i * P.n_vars + P.genes[g].var]; // extractActiveVariables
            fitness = fit[i] + goal_fitness_secondary(P, gp, (const double*)x, seed);
        }
        if(fitness < best_fitness)
        {
            best_fitness = fitness;
            best_index = i;
        }
    }
    if(best_fitness == DBLMAX)
        for(int i = 0; i < islands; i++)
            if(fit[i] < best_fitness)
            {
                best_fitness = fit[i];
                best_index = i;
            }
    *best = best_fitness;
    return best_index;
}

// ---------------------------------------------------------------------------
// reproduce() for one child, src/ik_evolution_2.cpp:263-301.
//   g0 = parent genes, gr0/gr1 = the two parents' gradients, rr = this child's gaussian
//   slab, rate_exp = fast_random_index(16) of this child.
// ---------------------------------------------------------------------------
BIOIK_HD void reproduce_child(const DProblem& P, int child_index, int rate_exp, const double* rr, const double* g0, const double* gr0, const double* gr1, double* child_genes, double* child_grads)
{
    double mutation_rate = (double)(1 << rate_exp) * (1.0 / (double)(1 << 23)); // :265
    double fmix = (child_index % 2 == 0) ? 0.2 : 0.0;                           // :268  (bool * 0.2)
    double gradient_factor = (double)(child_index % 3);                        // :269
    for(int i = 0; i < P.n; i++)
    {
        const DGene& Gn = P.genes[i];
        double r = rr[i];
        double f = mutation_rate * Gn.span;
        double gene = g0[i];
        double parent_gene = gene;
        gene += r * f;
        double parent_gradient = mix(gr0[i], gr1[i], fmix);
        double gradient = parent_gradient * gradient_factor;
        gene += gradient;
        gene = clampd(gene, Gn.clip_min, Gn.clip_max);
        child_genes[i] = gene;
        if(child_grads) child_grads[i] = mix(parent_gradient, gene - parent_gene, 0.3);
    }
    // :320-324 normalizeFast on the quaternion genes of floating joints (include/bio_ik/frame.h:231-238)
    for(int k = 0; k < P.n_quat; k++)
    {
        double* q = child_genes + P.quat_gene[k];
        const double f = (3.0 - (q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])) * 0.5;
        q[0] = q[0] * f, q[1] = q[1] * f, q[2] = q[2] * f, q[3] = q[3] * f;
    }
}

// ---------------------------------------------------------------------------
// RNG pieces that run on the device (src/ik_base.h:49-126)
// ---------------------------------------------------------------------------
// std::minstd_rand: x <- 48271 x mod 2147483647
BIOIK_HD uint32_t minstd_next(uint32_t& s)
{
    s = (uint32_t)(((uint64_t)s * 48271ull) % 2147483647ull);
    return s;
}
// std::uniform_real_distribution<double>(0,1)(minstd) = generate_canonical<double,53>: two draws
// (libstdc++ bits/random.tcc): sum = (a-1) + (b-1)*R, R = 2147483646; ret = sum / R^2
BIOIK_HD double minstd_uniform01(uint32_t& s)
{
    double a = (double)(minstd_next(s) - 1u);
    double b = (double)(minstd_next(s) - 1u);
    double sum = a * 1.0;           // __sum += (urng()-min) * __tmp, __tmp = 1
    sum = sum + b * 2147483646.0;   // __tmp = R
    double ret = sum / 4611686009837453316.0; // R*R rounded to double (4611686009837453316 = 2147483646^2 is exact below 2^63; double rounding below)
    if(ret >= 1.0) ret = 0.99999999999999989; // nextafter(1, 0)
    return ret;
}
// Random::random(min, max), src/ik_base.h:64
BIOIK_HD double minstd_random(uint32_t& s, double lo, double hi) { return minstd_uniform01(s) * (hi - lo) + lo; }
// std::uniform_int_distribution<size_t>(0, n-1)(minstd) for n-1 < 2147483645 (libstdc++ bits/uniform_int_dist.h, downscaling branch)
BIOIK_HD uint32_t minstd_index(uint32_t& s, uint32_t n)
{
    const uint64_t urngrange = 2147483645ull;
    uint64_t uerange = (uint64_t)n; // urange + 1
    uint64_t scaling = urngrange / uerange;
    uint64_t past = uerange * scaling;
    uint64_t ret;
    do
        ret = (uint64_t)minstd_next(s) - 1ull;
    while(ret >= past);
    return (uint32_t)(ret / scaling);
}

// ---------------------------------------------------------------------------
// Problem::checkSolutionActiveVariables, src/problem.cpp:259-341 (KDL semantics per
// SURVEY.md Appendix C).  Thresholds are compared against 1e-5-scale quantities; the
// libm-class functions here (atan2, acos, sqrt) are not part of the bit-exact contract.
// ---------------------------------------------------------------------------
BIOIK_HD void quat_to_matrix(const Q4& q, double* R)
{
    double x = q.x, y = q.y, z = q.z, w = q.w;
    double x2 = x * x, y2 = y * y, z2 = z * z, w2 = w * w;
    R[0] = w2 + x2 - y2 - z2; R[1] = 2 * x * y - 2 * w * z; R[2] = 2 * x * z + 2 * w * y;
    R[3] = 2 * x * y + 2 * w * z; R[4] = w2 - x2 + y2 - z2; R[5] = 2 * y * z - 2 * w * x;
    R[6] = 2 * x * z - 2 * w * y; R[7] = 2 * y * z + 2 * w * x; R[8] = w2 - x2 - y2 + z2;
}
BIOIK_HD void kdl_twist(const F7& fa, const F7& fb, double* vel, double* rot)
{
    double Ra[9], Rb[9], M[9];
    quat_to_matrix(fa.q, Ra);
    quat_to_matrix(fb.q, Rb);
    double d0 = fb.p.x - fa.p.x, d1 = fb.p.y - fa.p.y, d2 = fb.p.z - fa.p.z;
    for(int i = 0; i < 3; i++) vel[i] = Ra[0 + i] * d0 + Ra[3 + i] * d1 + Ra[6 + i] * d2;
    for(int i = 0; i < 3; i++)
        for(int j = 0; j < 3; j++) M[i * 3 + j] = Ra[0 + i] * Rb[0 + j] + Ra[3 + i] * Rb[3 + j] + Ra[6 + i] * Rb[6 + j];
    double ax = M[7] - M[5], ay = M[2] - M[6], az = M[3] - M[1];
    double sa = BIOIK_SQRT(ax * ax + ay * ay + az * az) * 0.5;
    double ca = (M[0] + M[4] + M[8] - 1.0) * 0.5;
    double angle = BIOIK_ATAN2(sa, ca);
    if(sa > 1e-12)
    {
        double f = angle / (2.0 * sa);
        rot[0] = ax * f; rot[1] = ay * f; rot[2] = az * f;
    }
    else if(ca > 0)
    {
        rot[0] = ax * 0.5; rot[1] = ay * 0.5; rot[2] = az * 0.5;
    }
    else
    {
        rot[0] = angle; rot[1] = 0; rot[2] = 0;
    }
}
BIOIK_HD bool all_below(const double* v, double eps) { return BIOIK_FABS(v[0]) < eps && BIOIK_FABS(v[1]) < eps && BIOIK_FABS(v[2]) < eps; }
BIOIK_HD double angle_shortest_path(const Q4& a, const Q4& b)
{
    double s = BIOIK_SQRT(qlen2(a.x, a.y, a.z, a.w) * qlen2(b.x, b.y, b.z, b.w));
    double d = a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
    if(d < 0) return BIOIK_ACOS((a.x * -b.x + a.y * -b.y + a.z * -b.z + a.w * -b.w) / s) * 2.0;
    return BIOIK_ACOS(d / s) * 2.0;
}
template <class AP, class AT, class AX, class AS> BIOIK_HD bool check_solution(const DProblem& P, AP gp, AT tips, AX x, AS seed)
{
    for(int gi = 0; gi < P.G; gi++)
    {
        const DGoal& g = P.goals[gi];
        if(g.secondary) continue;
        AP p = gp + gi * GOAL_NPARAM;
        F7 fb = load_frame(tips + 7 * g.tip);
        F7 fa;
        fa.p = V3{0, 0, 0};
        fa.q = Q4{0, 0, 0, 1};
        double vel[3], rot[3];
        if(g.type == G_POSITION)
        {
            fa.p = V3{p[0], p[1], p[2]};
            if(P.dpos != DBLMAX)
            {
                double pd = BIOIK_SQRT(len2(fb.p.x - fa.p.x, fb.p.y - fa.p.y, fb.p.z - fa.p.z));
                if(!(pd <= P.dpos)) return false;
            }
            if(P.dtwist != DBLMAX)
            {
                kdl_twist(fa, fb, vel, rot);
                if(!all_below(vel, P.dtwist)) return false;
            }
        }
        else if(g.type == G_ORIENTATION)
        {
            fa.q = Q4{p[3], p[4], p[5], p[6]};
            if(P.drot != DBLMAX)
            {
                double rd = angle_shortest_path(fb.q, fa.q) * 180 / 3.14159265358979323846;
                if(!(rd <= P.drot)) return false;
            }
            if(P.dtwist != DBLMAX)
            {
                kdl_twist(fa, fb, vel, rot);
                if(!all_below(rot, P.dtwist)) return false;
            }
        }
        else if(g.type == G_POSE)
        {
            fa.p = V3{p[0], p[1], p[2]};
            fa.q = Q4{p[3], p[4], p[5], p[6]};
            if(P.dpos != DBLMAX || P.drot != DBLMAX)
            {
                double pd = BIOIK_SQRT(len2(fb.p.x - fa.p.x, fb.p.y - fa.p.y, fb.p.z - fa.p.z));
                double rd = angle_shortest_path(fb.q, fa.q) * 180 / 3.14159265358979323846;
                if(!(pd <= P.dpos)) return false;
                if(!(rd <= P.drot)) return false;
            }
            if(P.dtwist != DBLMAX)
            {
                kdl_twist(fa, fb, vel, rot);
                if(!all_below(vel, P.dtwist) || !all_below(rot, P.dtwist)) return false;
            }
        }
        else
        {
            double dmax = BIOIK_FMIN(BIOIK_FMIN(DBLMAX, P.dpos), P.dtwist);
            double d = goal_value(P, g, p, tips, x, seed) * g.weight_sq;
            if(!(d < dmax * dmax)) return false;
        }
    }
    return true;
}

} // namespace bioik
