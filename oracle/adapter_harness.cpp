// adapter_harness.cpp — compiles adapter/ik_evolution_2_b200.cpp INSIDE the reference's own solver framework
// (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
//
// One translation unit = the reference's src/ik_evolution_2.cpp + src/problem.cpp + src/ik_parallel.h where they lie under
// the reference checkout (through ref_harness.cpp and the stand-in third-party headers of oracle/shims/, nothing copied) + the
// adapter exactly as a bio_ik maintainer would add it.  It is linked against libbioik_b200.so and exports the entry points
// the `-m gpu` tests of tests/test_adapter.py call, so that
//   * IKFactory::create("bio2_memetic_b200", params) -> initialize(problem) -> step() x k -> getSolution() runs through the
//     reference's own types (IKBase, Problem, GoalInfo, the goal classes), and
//   * IKParallel::solve (src/ik_parallel.h:148-269) - the reference's driver, its thread pool on the boost::barrier shim,
//     its own exact FK + checkSolution on what the adapter returns - drives the GPU solver unchanged.
// Built by `make -C oracle adapter` into oracle/_ref/libbioik_adapter.so (git-ignored, travels to the GPU box).
#include <chrono>
#include "ref_harness.cpp"

#include "ik_parallel.h"

#include "../adapter/ik_evolution_2_b200.cpp"

namespace
{
struct AdapterCase
{
    std::shared_ptr<moveit::core::RobotModel> model;
    moveit::core::JointModelGroup group;
    IKParams params;
    GoalSet goals;
    Problem problem;
};

// robot + joint group + goals + Problem::initialize, all through the reference's public API (as ref_solve_batch does)
void makeCase(AdapterCase& c, const BioikRobot* robot, const BioikProblem* problem, const char* solver, int random_seed, int thread_count, const double* goal_params, const double* seed)
{
    c.model = makeRobot(robot);
    c.group.parent_ = c.model.get();
    for(int i = 0; i < problem->n_active; i++)
    {
        c.group.variable_names_.push_back(c.model->variable_names_[problem->active_vars[i]]);
        auto* joint = c.model->joint_of_variable_[problem->active_vars[i]];
        if(c.group.active_joints_.empty() || c.group.active_joints_.back() != joint) c.group.active_joints_.push_back(joint);
    }
    IKParams& params = c.params;
    params.robot_model = c.model;
    params.joint_model_group = &c.group;
    params.solver_class_name = solver;
    params.enable_counter = false;
    params.thread_count = thread_count;
    params.random_seed = random_seed;
    params.dpos = problem->dpos, params.drot = problem->drot, params.dtwist = problem->dtwist;
    params.opt_no_wipeout = false, params.population_size = 8, params.elite_count = 4, params.linear_fitness = false;
    makeGoals(*c.model, problem, goal_params, c.goals);
    c.problem.initial_guess.assign(seed, seed + robot->n_vars);
    c.problem.timeout = 0;
    c.problem.initialize(c.model, &c.group, params, c.goals.ptrs, nullptr);
    if(c.problem.active_variables.size() != (size_t)problem->n_active || c.problem.tip_link_indices.size() != (size_t)problem->n_tips) throw std::runtime_error("Problem::initialize disagrees with the flattened problem (sizes)");
    for(int i = 0; i < problem->n_active; i++)
        if((int)c.problem.active_variables[i] != problem->active_vars[i]) throw std::runtime_error("Problem::initialize disagrees with the flattened problem (active variable order)");
}
} // namespace

extern "C" {

// 1 if IKFactory knows the solver class `name` AND can construct it (needs a CUDA device for the *_b200 classes); else 0 with
// the exception text in ref_last_error()
int adapter_can_create(const BioikRobot* robot, const BioikProblem* problem, const char* name, const double* seed)
{
    try
    {
        AdapterCase c;
        makeCase(c, robot, problem, name, 1, 1, nullptr, seed);
        std::unique_ptr<IKSolver> s(IKFactory::create(name, c.params));
        return 1;
    }
    catch(std::exception& e)
    {
        g_error = e.what();
        return 0;
    }
}

// IKFactory::create(solver) -> initialize(problem) -> step() x steps -> getSolution(), optionally on a clone made by
// IKFactory::clone (the copy constructor IKParallel uses for its extra threads), and twice in a row on the same object
// (a plugin instance re-initialises its solver for every query).  out_solutions: [n_queries][n_vars].
int adapter_steps(const BioikRobot* robot, const BioikProblem* problem, const char* solver, int random_seed, int n_queries, const double* goal_params, const double* seeds, int steps, int use_clone, double* out_solutions)
{
    try
    {
        const size_t per_gp = (size_t)problem->n_goals * BIOIK_GOAL_NPARAM;
        AdapterCase c0;
        makeCase(c0, robot, problem, solver, random_seed, 1, goal_params, seeds);
        std::unique_ptr<IKSolver> first(IKFactory::create(solver, c0.params));
        std::unique_ptr<IKSolver> copy;
        IKSolver* s = first.get();
        if(use_clone)
        {
            copy.reset(IKFactory::clone(first.get()));
            first.reset(); // the clone must not depend on the object it was copied from
            s = copy.get();
        }
        s->thread_index = 0;
        for(int q = 0; q < n_queries; q++)
        {
            AdapterCase c;
            makeCase(c, robot, problem, solver, random_seed, 1, goal_params ? goal_params + q * per_gp : nullptr, seeds + (size_t)q * robot->n_vars);
            s->canceled = false; // IKParallel::solve does this before every solve (src/ik_parallel.h:211-212)
            s->initialize(c.problem);
            for(int k = 0; k < steps; k++) s->step();
            const std::vector<double>& r = s->getSolution();
            std::copy(r.begin(), r.end(), out_solutions + (size_t)q * robot->n_vars);
        }
        return 0;
    }
    catch(std::exception& e)
    {
        g_error = e.what();
        return 1;
    }
}

// The reference's driver, unchanged: IKParallel(params) -> initialize(problem) -> solve() with a wall-clock timeout.
// out_iterations = IKParallel::iteration_count (one per 4-step burst, src/ik_parallel.h:167).
int adapter_parallel(const BioikRobot* robot, const BioikProblem* problem, const char* solver, int random_seed, int thread_count, const double* goal_params, const double* seed, double timeout_seconds, double* out_solution,
                     int32_t* out_success, double* out_fitness, int32_t* out_iterations)
{
    try
    {
        AdapterCase c;
        makeCase(c, robot, problem, solver, random_seed, thread_count, goal_params, seed);
        IKParallel ik(c.params);
        c.problem.timeout = ros::WallTime::now().toSec() + timeout_seconds;
        ik.initialize(c.problem);
        ik.solve();
        const std::vector<double>& r = ik.getSolution();
        std::copy(r.begin(), r.end(), out_solution);
        if(out_success) *out_success = ik.getSuccess() ? 1 : 0;
        if(out_fitness) *out_fitness = ik.getSolutionFitness();
        if(out_iterations) *out_iterations = (int32_t)ik.iteration_count;
        // ~ParallelExecutor (src/ik_parallel.h:80-86) sets `exit` and then meets its workers at the barrier, assuming they are back at
        // the top of their loop.  A worker that has not yet passed the `if(exit) break;` after the END barrier of run() (:67-68)
        // would leave instead and the destructor would wait forever - a teardown race of the reference that a long-lived plugin
        // never meets, but a harness destroying the driver microseconds after solve() does.  Give the workers time to loop around.
        if(thread_count > 1) std::this_thread::sleep_for(std::chrono::milliseconds(50));
        return 0;
    }
    catch(std::exception& e)
    {
        g_error = e.what();
        return 1;
    }
}
}
