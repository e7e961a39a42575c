/*
 * bioik_b200.h — C ABI of libbioik_b200.so: the H100-native bio2 / bio2_memetic
 * population loop of TAMS-Group/bio_ik, evaluated for whole batches of
 * independent IK queries on one GPU.
 *
 * This is the drop-in boundary of SURVEY.md §8(b).  Every entry point names the
 * reference interface it replaces (paths relative to the reference tree).
 * Plain pointers and sizes only; no C++/torch/CUDA types cross this header.
 * All functions return a BIOIK_* status and never throw across the ABI;
 * bioik_last_error() returns a human-readable message for the last failure.
 *
 * There is NO CPU fallback behind this ABI: every compute entry point launches
 * sm_90a kernels and fails with BIOIK_E_CUDA if no usable device is present.
 */
#ifndef BIOIK_B200_H
#define BIOIK_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BIOIK_ABI_VERSION 2 /* 2: BioikRobot::link_mass / link_com, BIOIK_GOAL_BALANCE, bioik_begin / bioik_step / bioik_get_solution */

/* ---- status codes (reference: ERROR(...) -> std::runtime_error, src/utils.h:122-129) */
enum {
    BIOIK_OK = 0,
    BIOIK_E_INVALID = 1,          /* bad argument / inconsistent tables            */
    BIOIK_E_UNSUPPORTED_GOAL = 2, /* goal needs a host callback / FCL (JointFunction,
                                     LinkFunction, Touch): keep the stock CPU solver */
    BIOIK_E_UNSUPPORTED_JOINT = 3,
    BIOIK_E_CUDA = 4,             /* CUDA runtime error or no device                */
    BIOIK_E_NO_PROBLEM = 5,       /* solve called before bioik_set_problem          */
    BIOIK_E_LIMIT = 6             /* problem exceeds a compiled-in capacity         */
};

/* ---- joint types (moveit::core::JointModel::JointType as used by
 *      src/forward_kinematics.h:78-139) */
enum {
    BIOIK_JOINT_FIXED = 0,
    BIOIK_JOINT_REVOLUTE = 1,
    BIOIK_JOINT_PRISMATIC = 2,
    BIOIK_JOINT_FLOATING = 3, /* 7 variables: x y z qx qy qz qw */
    BIOIK_JOINT_PLANAR = 4    /* 3 variables: x y theta         */
};

/* ---- goal types: the closed-form goal classes of include/bio_ik/goal_types.h.
 *      p[] layout per type is given beside each enumerator.  Quaternions are
 *      (x,y,z,w) and must already be normalised the way the reference
 *      constructors/setters do it (goal_types.h:110,114,139,146). */
enum {
    BIOIK_GOAL_POSITION = 1,             /* goal_types.h:96      p[0..2]=position                       */
    BIOIK_GOAL_ORIENTATION = 2,          /* goal_types.h:115-119 p[3..6]=orientation                    */
    BIOIK_GOAL_POSE = 3,                 /* goal_types.h:149-180 p[0..2],p[3..6],p[7]=rotation_scale    */
    BIOIK_GOAL_LOOK_AT = 4,              /* goal_types.h:204-211 p[0..2]=axis p[3..5]=target            */
    BIOIK_GOAL_MAX_DISTANCE = 5,         /* goal_types.h:235-240 p[0..2]=target p[3]=distance           */
    BIOIK_GOAL_MIN_DISTANCE = 6,         /* goal_types.h:264-269 p[0..2]=target p[3]=distance           */
    BIOIK_GOAL_LINE = 7,                 /* goal_types.h:293-297 p[0..2]=position p[3..5]=direction     */
    BIOIK_GOAL_PLANE = 8,                /* goal_types.h:321-327 p[0..2]=position p[3..5]=normal        */
    BIOIK_GOAL_AVOID_JOINT_LIMITS = 9,   /* goal_types.h:387-401 (no params)                            */
    BIOIK_GOAL_CENTER_JOINTS = 10,       /* goal_types.h:412-425 (no params)                            */
    BIOIK_GOAL_REGULARIZATION = 11,      /* goal_types.h:435-444 (no params)                            */
    BIOIK_GOAL_MINIMAL_DISPLACEMENT = 12,/* goal_types.h:455-465 (no params)                            */
    BIOIK_GOAL_JOINT_VARIABLE = 13,      /* goal_types.h:494-498 var=robot variable, p[0]=position      */
    BIOIK_GOAL_SIDE = 14,                /* goal_types.h:606-613 p[0..2]=axis p[3..5]=direction         */
    BIOIK_GOAL_DIRECTION = 15,           /* goal_types.h:637-643 p[0..2]=axis p[3..5]=direction         */
    BIOIK_GOAL_CONE = 16,                /* goal_types.h:700-711 p[0..2]=position p[3]=position_weight
                                                                 p[4..6]=axis p[7..9]=direction p[10]=angle */
    BIOIK_GOAL_BALANCE = 17              /* goal_types.h:540-568, src/goal_types.cpp:231-272  p[0..2]=target p[3..5]=axis.
                                            Centre of mass over every link with BioikRobot::link_mass > 0; those links must
                                            be tip links of the problem, in link order (what BalanceGoal::describe adds). */
};

#define BIOIK_GOAL_NPARAM 12

/* Flattened moveit::core::RobotModel (SURVEY.md Appendix B).  One parent joint
 * per link; joint arrays are indexed by the joint's child link.  Links must be
 * ordered parents-before-children.  Replaces what RobotJointEvaluator /
 * RobotFK_Fast_Base / RobotInfo read from MoveIt
 * (src/forward_kinematics.h:192-213,230-246; include/bio_ik/robot_info.h:70-105). */
typedef struct BioikRobot {
    int32_t n_links;
    int32_t n_vars;
    const int32_t* link_parent;      /* [n_links] parent link, -1 for the root                      */
    const int32_t* joint_type;       /* [n_links] BIOIK_JOINT_*                                     */
    const int32_t* joint_first_var;  /* [n_links] first variable index (-1 if the joint has none)   */
    const double* link_origin;       /* [n_links][7] getJointOriginTransform(): px py pz qx qy qz qw */
    const double* joint_axis;        /* [n_links][3] revolute / prismatic axis                      */
    const int32_t* joint_mimic;      /* [n_links] child link of the mimicked joint, -1 if none      */
    const double* joint_mimic_factor;/* [n_links]                                                   */
    const double* joint_mimic_offset;/* [n_links]                                                   */
    const double* var_min;           /* [n_vars] VariableBounds::min_position_                      */
    const double* var_max;           /* [n_vars] VariableBounds::max_position_                      */
    const int32_t* var_bounded;      /* [n_vars] VariableBounds::position_bounded_                  */
    const double* var_max_velocity;  /* [n_vars] VariableBounds::max_velocity_                      */
    /* URDF inertials, read only by BalanceGoal (src/goal_types.cpp:236-250); NULL = no link has mass */
    const double* link_mass;         /* [n_links] urdf::Link::inertial->mass (0 = none)             */
    const double* link_com;          /* [n_links][3] urdf::Link::inertial->origin.position          */
} BioikRobot;

/* Flattened GoalInfo (src/problem.h:121-130; field set of the older struct at
 * src/problem.h:91-117). */
typedef struct BioikGoal {
    int32_t type;      /* BIOIK_GOAL_*                                                          */
    int32_t tip;       /* index into BioikProblem::tip_links (link goals), else 0               */
    int32_t secondary; /* GoalContext::goal_secondary_                                          */
    int32_t var;       /* JOINT_VARIABLE: robot variable index                                  */
    double weight;     /* GoalContext::goal_weight_  (fitness uses weight*weight)               */
    double p[BIOIK_GOAL_NPARAM]; /* default parameters; per-query values override them in solve */
} BioikGoal;

/* Flattened Problem (src/problem.h:131-136, built by src/problem.cpp:72-228). */
typedef struct BioikProblem {
    int32_t n_tips;
    const int32_t* tip_links;   /* [n_tips] Problem::tip_link_indices                      */
    int32_t n_active;
    const int32_t* active_vars; /* [n_active] Problem::active_variables (gene order)       */
    int32_t n_goals;
    const BioikGoal* goals;     /* primary and secondary goals in Problem order            */
    double dpos, drot, dtwist;  /* IKParams thresholds, src/problem.cpp:90-95 (DBL_MAX=off) */
} BioikProblem;

/* Solver constants the reference hard-codes (src/ik_evolution_2.cpp:137-138,
 * 349-351,453) exposed as parameters (SURVEY.md D2). */
typedef struct BioikSolverCfg {
    int32_t population;    /* children.size() = 2 parents + child_count; reference 18   */
    int32_t generations;   /* per species per step(): reference 8 (memetic) / 16        */
    int32_t memetic;       /* 0 = bio2, 'q' = bio2_memetic, 'l' = bio2_memetic_l        */
    int32_t memetic_iters; /* reference 8                                               */
    uint32_t table_seed;   /* IKParams::random_seed: seeds the two shared 8Mi lookup
                              tables exactly like Random::Random (src/ik_base.h:118-125) */
    int32_t device;        /* CUDA device ordinal                                       */
} BioikSolverCfg;

typedef struct bioik_ctx bioik_ctx;

/* IKFactory::create(name, params) + IKBase ctor (src/ik_parallel.h:119,
 * src/ik_base.h:144-151): builds the solver context, uploads the robot table and
 * the two RNG lookup tables to HBM. */
int bioik_create(const BioikRobot* robot, const BioikSolverCfg* cfg, bioik_ctx** out);
void bioik_destroy(bioik_ctx* ctx);

/* IKBase::initialize(problem) + IKEvolution2::initialize structure part
 * (src/ik_base.h:154-161, src/ik_evolution_2.cpp:111-230): link schedule, gene
 * limits, goal table.  Per-query data (targets, seeds) arrive with solve. */
int bioik_set_problem(bioik_ctx* ctx, const BioikProblem* problem);

/* The batch form of IKParallel::solve -> solverthread (src/ik_parallel.h:148-269)
 * around IKEvolution2::step (src/ik_evolution_2.cpp:328-646) with the timeout
 * replaced by a step budget (SURVEY.md §8(c) batch contract):
 *   query q starts as a freshly constructed solver sharing the lookup tables,
 *   rng = minstd_rand(rng_seeds[q]), runs `steps` step()s; success is tested on
 *   getSolution() after every 4th step (the driver's 4-step bursts,
 *   src/ik_parallel.h:165-181) and after the last step; with
 *   early_exit != 0 a query stops at its first successful test, like the
 *   reference driver.
 * Host pointers; H2D/D2H copies are part of the call.
 *   goal_params   [B][n_goals][BIOIK_GOAL_NPARAM] or NULL (use BioikGoal::p)
 *   seeds         [B][n_vars]  Problem::initial_guess (full variable vector)
 *   rng_seeds     [B]
 *   out_solutions [B][n_vars]  IKSolver::getSolution()
 *   out_fitness   [B]          primary fitness of the solution (ik_parallel.h:181)
 *   out_success   [B]          Problem::checkSolutionActiveVariables of the solution
 *   out_steps     [B]          step() calls executed for the query                   */
int bioik_solve_batch(bioik_ctx* ctx, int32_t B, const double* goal_params, const double* seeds,
                      const uint32_t* rng_seeds, int32_t steps, int32_t early_exit,
                      double* out_solutions, double* out_fitness, int32_t* out_success,
                      int32_t* out_steps);

/* Same, all buffers already resident in device memory of ctx's device; work is
 * enqueued on `cuda_stream` (a cudaStream_t passed as void*, NULL = the context's
 * own stream) and NOT synchronised. */
int bioik_solve_batch_device(bioik_ctx* ctx, int32_t B, const double* d_goal_params,
                             const double* d_seeds, const uint32_t* d_rng_seeds, int32_t steps,
                             int32_t early_exit, double* d_out_solutions, double* d_out_fitness,
                             int32_t* d_out_success, int32_t* d_out_steps, void* cuda_stream);

/* Block until the context's stream has drained. */
int bioik_synchronize(bioik_ctx* ctx);

/* ---- component entry points (used by the parity tests; same kernels) -------- */

/* RobotFK_Fast_Base::applyConfiguration (src/forward_kinematics.h:331-354) for a
 * batch of full variable vectors [B][n_vars] -> tip frames [B][n_tips][7]. */
int bioik_fk_batch(bioik_ctx* ctx, int32_t B, const double* variables, double* out_tip_frames);

/* RobotFK_Jacobian::computeJacobian + RobotFK_Mutator::initializeMutationApproximator
 * (src/forward_kinematics.h:600-730,802-930) at [B][n_vars] base points ->
 * delta frames [B][n_tips][n_active][7] (pos xyz, rot xyzw). */
int bioik_approx_batch(bioik_ctx* ctx, int32_t B, const double* variables, double* out_delta_frames);

/* computeApproximateMutations + computeFitnessActiveVariables
 * (src/forward_kinematics.h:1061-1233, src/ik_base.h:167-185) at base points
 * [B][n_vars] for genotypes [B][M][n_active] -> primary and secondary fitness
 * [B][M] each (either output may be NULL). */
int bioik_approx_fitness_batch(bioik_ctx* ctx, int32_t B, int32_t M, const double* goal_params,
                               const double* seeds, const double* base_variables,
                               const double* genotypes, double* out_primary, double* out_secondary);

/* Solver state after `steps` steps, for trajectory-level parity:
 *   out_genes     [B][2 species][2 individuals][n_active]
 *   out_gradients [B][2][2][n_active]
 *   out_species_fitness [B][2]   (array order, i.e. after the species sort)     */
int bioik_solve_batch_trace(bioik_ctx* ctx, int32_t B, const double* goal_params,
                            const double* seeds, const uint32_t* rng_seeds, int32_t steps,
                            double* out_genes, double* out_gradients,
                            double* out_species_fitness, double* out_solutions,
                            double* out_fitness);

/* Options of a solver context.
 * BIOIK_OPT_REFERENCE_STALE_TIPS (default 0): 1 reproduces quirk Q2 of the reference's memetic step on problems where some
 *   variable cannot move some tip.  RobotFK_Mutator::computeApproximateMutation1 skips such tips
 *   (src/forward_kinematics.h:940), so the gradient probe (src/ik_evolution_2.cpp:469-470) scores them on whatever
 *   phenotypes3[0] held before - the write of an earlier probe, or the frames of the last f3 evaluation (:494) of the previous
 *   iteration / species / step; a fresh reference solver reads uninitialised memory there, this library starts from
 *   identity frames.  With 0 the probe scores those tips on the unmoved frame (out[t] = in[t], the evident intent).
 *   Single-chain problems (every variable moves every tip) are unaffected.
 * BIOIK_OPT_ISLAND_STREAM_STRIDE (default 0): the islands of a query (bioik_begin / bioik_solve_islands with islands > 1) are,
 *   like IKParallel's threads (src/ik_parallel.h:84-86, src/utils.h:423: clones of one solver, SURVEY.md Q3), replicas that replay
 *   ONE sequence of gaussians / rate exponents / fast_random values and differ only through their minstd_rand seeds (wipe-out
 *   re-rolls, pre-selection counts).  A value k > 0 starts island i `i * k` solver steps into that sequence, so the islands
 *   mutate differently from their first generation; island 0 and every plain batch are unaffected.  Results are then not those of
 *   the reference's clone islands (the oracle restates the option; tests/test_islands.py). */
enum { BIOIK_OPT_REFERENCE_STALE_TIPS = 1, BIOIK_OPT_ISLAND_STREAM_STRIDE = 2 };
int bioik_set_option(bioik_ctx* ctx, int32_t option, int32_t value);

/* IKBase::canceled (src/ik_base.h:143; set for every solver when the driver finishes or times out, polled in the solver's
 * loops, src/ik_evolution_2.cpp:355,457): makes every run of the solve that is in flight count as finished from the next
 * kernel on; the call returns what the runs had reached.  The one entry point that may be called from another thread
 * while a solve is running; every bioik_solve_* call and bioik_begin clear the flag when they start (IKParallel::solve resets
 * canceled at the start of each solve, src/ik_parallel.h:211-212). */
int bioik_cancel(bioik_ctx* ctx);

/* One MoveIt-style query solved by many differently seeded islands at once, then reduced the way the reference
 * reduces its solver threads (SURVEY.md §8(f) rows 1 and 3):
 *   - run q * islands + k is island k of query q: the query's goal parameters and seed, rng_seeds[q * islands + k];
 *     the reference's IKParallel starts identical clones on every thread (src/ik_parallel.h:119-127) - the island
 *     seeds are what makes the extra runs worth something;
 *   - selection = IKParallel::solve (src/ik_parallel.h:218-258): among the successful islands the smallest
 *     primary (+ secondary, when the problem has secondary goals) fitness, else the smallest primary fitness;
 *     first island wins ties;
 *   - early_exit: 0 = every island runs `steps` steps; 1 = an island stops at its own first successful test; 2 = like
 *     the reference's driver, whose `finished` flag makes every solver thread leave its loop once one of them has
 *     passed the test (src/ik_parallel.h:160-186): all islands of a query stop after the 4-step check at which the
 *     first of them succeeded (deterministic: the islands run in lock step);
 *   - wrap != 0 applies the plugin's angle wrap to the selected solution (src/kinematics_plugin.cpp:580-611):
 *     revolute variables of robots without mimic joints are moved by multiples of 2 pi next to the seed, wrapped
 *     inside [min, max] and clamped.  (MoveIt's enforcePositionBounds, :614, is MoveIt code and not applied.)
 * Host pointers.
 *   goal_params   [Q][n_goals][BIOIK_GOAL_NPARAM] or NULL      seeds       [Q][n_vars]
 *   rng_seeds     [Q * islands]
 *   out_solutions [Q][n_vars]   out_fitness [Q] (IKParallel::getSolutionFitness: incl. secondary when successful)
 *   out_success   [Q]           out_island  [Q] index of the selected island   out_steps [Q] its step() calls
 * Any output except out_solutions may be NULL. */
int bioik_solve_islands(bioik_ctx* ctx, int32_t Q, int32_t islands, const double* goal_params, const double* seeds,
                        const uint32_t* rng_seeds, int32_t steps, int32_t early_exit, int32_t wrap,
                        double* out_solutions, double* out_fitness, int32_t* out_success, int32_t* out_island,
                        int32_t* out_steps);

/* ---- the resumable form: the reference's solver interface initialize / step / getSolution -----------------------------
 * IKParallel::solverthread drives a solver through exactly these three calls (src/ik_parallel.h:156,165-181):
 *   solvers[i]->initialize(problem);  solvers[i]->step() x4;  result = solvers[i]->getSolution();  ... until success/timeout.
 * bioik_begin / bioik_step / bioik_get_solution are those calls for Q queries x `islands` differently seeded runs each;
 * the solver state stays resident on the device between the calls, so k calls of bioik_step(ctx, 1) cost the same device
 * work as one bioik_step(ctx, k).  bioik_solve_islands is begin + step(4) ... + get_solution.
 * adapter/ik_evolution_2_b200.cpp is the IKBase subclass that forwards to them. */

/* IKBase::initialize(problem) + IKEvolution2::initialize (src/ik_base.h:154-161, src/ik_evolution_2.cpp:111-230) for every
 * run: copies goal_params [Q][n_goals][BIOIK_GOAL_NPARAM] (or NULL), seeds [Q][n_vars] and rng_seeds [Q * islands] to the
 * device (the host buffers are free when the call returns) and resets genes, gradients, species, solution and RNG state.
 * max_steps > 0: a step budget - like bioik_solve_islands the driver's test then also runs after the last step and
 * bioik_step never goes beyond it; 0: no budget (the reference's wall-clock loop: the caller decides when to stop).
 * early_exit as in bioik_solve_islands. */
int bioik_begin(bioik_ctx* ctx, int32_t Q, int32_t islands, const double* goal_params, const double* seeds,
                const uint32_t* rng_seeds, int32_t max_steps, int32_t early_exit);

/* IKBase::step() (src/ik_evolution_2.cpp:328-646) `nsteps` times for every run that is still going; returns when the
 * device has finished them.  out_active (may be NULL) receives the number of runs that would execute a further step
 * (0 once every run has finished through its early exit, the budget or bioik_cancel). */
int bioik_step(bioik_ctx* ctx, int32_t nsteps, int32_t* out_active);

/* IKBase::getSolution() of every run, then what the reference's driver derives from it: exact FK + checkSolution +
 * computeFitness per run (src/ik_parallel.h:173-181) and the selection among the runs of a query
 * (src/ik_parallel.h:218-258); outputs as in bioik_solve_islands.  May be called after any bioik_step and does not
 * disturb the solve. */
int bioik_get_solution(bioik_ctx* ctx, int32_t wrap, double* out_solutions, double* out_fitness, int32_t* out_success,
                       int32_t* out_island, int32_t* out_steps);

/* The result slab of a multi-GPU gather (SURVEY.md §8(e): one all-gather of the per-GPU results per solve round): packs the four
 * device-resident outputs of bioik_solve_batch_device into d_slab [B][n_vars + 3] = solution | fitness | success | steps
 * (all float64) on `cuda_stream`, not synchronised.  bio_ik_b200/distributed.py hands that slab to NCCL. */
int bioik_pack_results_device(bioik_ctx* ctx, int32_t B, const double* d_solutions, const double* d_fitness,
                              const int32_t* d_success, const int32_t* d_steps, double* d_slab, void* cuda_stream);

/* Template instantiation of the kernel that bioik_kernel_time reports as the generation kernel for the solve shape last used
 * (e.g. "k_persist<1, 4, 1, false, 7, false, 16, true, false>"); "" before the first solve. */
const char* bioik_kernel_name(const bioik_ctx* ctx);

/* Number of kernel launches issued by this context so far (bench.py gpu_launches). */
int64_t bioik_launch_count(const bioik_ctx* ctx);

/* Device-time of the dominant (generation) kernel and of the serial kernels accumulated
 * since the last call with reset != 0, measured with CUDA events on the launching
 * stream; returns milliseconds and the number of launches through the out parameters.
 * Per-launch timing is switched on by the first call (reset 0 or 1) and off again by
 * reset == 2; while it is off, repeated bioik_solve_batch calls of one shape replay a
 * CUDA graph. */
int bioik_kernel_time(bioik_ctx* ctx, int32_t reset, double* out_ms_evolve, int64_t* out_launches_evolve,
                      double* out_ms_serial, int64_t* out_launches_serial);

const char* bioik_last_error(const bioik_ctx* ctx); /* ctx may be NULL: create() errors */
int bioik_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* BIOIK_B200_H */
