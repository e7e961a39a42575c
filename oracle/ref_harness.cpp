// ref_harness.cpp — builds the REFERENCE's own bio2 solver (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
//
// This translation unit #includes the reference's sources where they lie in the reference checkout (REFERENCE= in oracle/Makefile)
// (src/ik_evolution_2.cpp, src/problem.cpp and everything they include) — nothing is copied into this
// repository — against the stand-in third-party headers of oracle/shims/.  It exposes the same batch
// entry point as the oracle so that
//   * tests can PIN the oracle restatement against the reference's real code (bit-for-bit, with the oracle
//     switched to libm sin/cos like the reference), and
//   * bench.py can time the reference's own CPU implementation ("kind": "reference").
// Batch contract (DESIGN.md §2): one solver is created through the reference's IKFactory (which fills the two
// static lookup tables from table_seed exactly as Random::Random does), every query runs on a copy-constructed
// clone of it (IKFactory::clone, the reference's own island mechanism) whose minstd engine is re-seeded with
// rng_seeds[q], and step() is called a fixed number of times.
// Goals are built through the reference's public constructors / setters only.  Several of them normalise their
// argument (goal_types.h:110,139,286,314); ref_effective_goal_params() returns the numbers the reference really
// stores, and the pinning tests hand exactly those to the oracle.
#include <algorithm>
#include <atomic>
#include <cfloat>
#include <cmath>
#include <csignal>
#include <functional>
#include <iostream>
#include <map>
#include <memory>
#include <mutex>
#include <random>
#include <set>
#include <sstream>
#include <stdexcept>
#include <string>
#include <thread>
#include <typeindex>
#include <unordered_map>
#include <unordered_set>
#include <vector>
#include <malloc.h>
#include <stdlib.h>
#include <emmintrin.h>
#include <immintrin.h>
#include <x86intrin.h>
#include "bioik_oracle.hpp" // only for det_sincos / det_acos (the arithmetic contract's sin, cos, acos)

// Test switch: with ref_set_contract_math(1) the two unqualified calls cos(half_angle) / sin(half_angle) of the
// reference's getJointFrame (forward_kinematics.h:103-104) resolve to these functions instead of libm's, and ConeGoal's
// acos goes through the shim hook - the reference then computes with the arithmetic contract of DESIGN.md §3 and can be
// compared with the CUDA path directly, bit for bit.  Default (0): libm, i.e. the reference exactly as it is.
namespace bio_ik
{
static int g_contract_math = 0;
inline double sin(double x)
{
    if(!g_contract_math) return ::sin(x);
    double s, c;
    bioik_oracle::det_sincos(x, &s, &c);
    return s;
}
inline double cos(double x)
{
    if(!g_contract_math) return ::cos(x);
    double s, c;
    bioik_oracle::det_sincos(x, &s, &c);
    return c;
}
}

#include "ik_evolution_2.cpp"
#include "problem.cpp"
#include "goal_types.cpp" // BalanceGoal::describe / evaluate (TouchGoal is compiled out, as with FCL >= 0.6)

#include "../include/bioik_b200.h"

#include <atomic>
#include <thread>

using namespace bio_ik;

namespace
{
thread_local std::string g_error;

std::shared_ptr<moveit::core::RobotModel> makeRobot(const BioikRobot* r)
{
    using namespace moveit::core;
    auto m = std::make_shared<RobotModel>();
    for(int l = 0; l < r->n_links; l++)
    {
        std::unique_ptr<JointModel> j;
        switch(r->joint_type[l])
        {
        case BIOIK_JOINT_REVOLUTE: j.reset(new RevoluteJointModel()), j->type_ = JointModel::REVOLUTE, j->variable_count_ = 1; break;
        case BIOIK_JOINT_PRISMATIC: j.reset(new PrismaticJointModel()), j->type_ = JointModel::PRISMATIC, j->variable_count_ = 1; break;
        case BIOIK_JOINT_FIXED: j.reset(new FixedJointModel()), j->type_ = JointModel::FIXED, j->variable_count_ = 0; break;
        case BIOIK_JOINT_FLOATING: j.reset(new JointModel()), j->type_ = JointModel::FLOATING, j->variable_count_ = 7; break; // handled by the reference itself (forward_kinematics.h:120-127)
        case BIOIK_JOINT_PLANAR: j.reset(new JointModel()), j->type_ = JointModel::PLANAR, j->variable_count_ = 3; break; // through the shim's computeTransform (forward_kinematics.h:128-135)
        default: throw std::runtime_error("ref harness: unknown joint type");
        }
        j->name_ = "joint" + std::to_string(l);
        j->joint_index_ = l;
        j->first_variable_index_ = r->joint_first_var[l] >= 0 ? r->joint_first_var[l] : 0;
        j->axis_ = Eigen::Vector3d(r->joint_axis[3 * l], r->joint_axis[3 * l + 1], r->joint_axis[3 * l + 2]);
        for(size_t k = 0; k < j->variable_count_; k++) j->variable_names_.push_back("var" + std::to_string(r->joint_first_var[l] + (int)k));
        std::unique_ptr<LinkModel> link(new LinkModel());
        link->name_ = "link" + std::to_string(l);
        link->link_index_ = l;
        const double* o = r->link_origin + 7 * l;
        link->joint_origin_transform_.t = Eigen::Vector3d(o[0], o[1], o[2]);
        link->joint_origin_transform_.R = Eigen::Quaterniond(o[6], o[3], o[4], o[5]).toRotationMatrix();
        m->links_.push_back(std::move(link));
        m->joints_.push_back(std::move(j));
    }
    m->variable_names_.resize(r->n_vars);
    m->bounds_.resize(r->n_vars);
    m->joint_of_variable_.assign(r->n_vars, nullptr);
    for(int l = 0; l < r->n_links; l++)
    {
        auto* link = m->links_[l].get();
        auto* joint = m->joints_[l].get();
        link->parent_joint_ = joint;
        joint->child_link_ = link;
        if(r->link_parent[l] >= 0)
        {
            link->parent_link_ = m->links_[r->link_parent[l]].get();
            joint->parent_link_ = link->parent_link_;
        }
        if(r->joint_mimic && r->joint_mimic[l] >= 0)
        {
            joint->mimic_ = m->joints_[r->joint_mimic[l]].get();
            joint->mimic_factor_ = r->joint_mimic_factor[l];
            joint->mimic_offset_ = r->joint_mimic_offset[l];
            m->mimic_joints_.push_back(joint);
        }
        {
            // URDF inertial of the link (read by BalanceGoal::describe only)
            auto ul = std::make_shared<urdf::Link>();
            if(r->link_mass && r->link_mass[l] != 0.0)
            {
                ul->inertial = std::make_shared<urdf::Inertial>();
                ul->inertial->mass = r->link_mass[l];
                if(r->link_com) ul->inertial->origin.position.x = r->link_com[3 * l], ul->inertial->origin.position.y = r->link_com[3 * l + 1], ul->inertial->origin.position.z = r->link_com[3 * l + 2];
            }
            m->urdf_->links_.emplace_back(link->name_, ul);
        }
        m->link_ptrs_.push_back(link);
        m->joint_ptrs_.push_back(joint);
        m->link_names_.push_back(link->name_);
        for(size_t k = 0; k < joint->variable_count_; k++)
        {
            int v = r->joint_first_var[l] + (int)k;
            m->variable_names_[v] = joint->variable_names_[k];
            m->joint_of_variable_[v] = joint;
            m->bounds_[v].min_position_ = r->var_min[v];
            m->bounds_[v].max_position_ = r->var_max[v];
            m->bounds_[v].position_bounded_ = r->var_bounded[v] != 0;
            m->bounds_[v].max_velocity_ = r->var_max_velocity[v];
        }
    }
    return m;
}

struct GoalSet
{
    std::vector<std::unique_ptr<Goal>> owned;
    std::vector<const Goal*> ptrs;
};

tf2::Vector3 V(const double* p) { return tf2::Vector3(p[0], p[1], p[2]); }

// reference goal objects from the flattened records, through the public API of include/bio_ik/goal_types.h
void makeGoals(const moveit::core::RobotModel& robot, const BioikProblem* pr, const double* gp, GoalSet& out)
{
    out.owned.clear(), out.ptrs.clear();
    for(int g = 0; g < pr->n_goals; g++)
    {
        const BioikGoal& bg = pr->goals[g];
        const double* p = gp ? gp + g * BIOIK_GOAL_NPARAM : bg.p;
        const std::string link = robot.link_names_[pr->tip_links[bg.tip]];
        const tf2::Quaternion q(p[3], p[4], p[5], p[6]);
        std::unique_ptr<Goal> goal;
        bool link_goal = true;
        switch(bg.type)
        {
        case BIOIK_GOAL_POSITION: goal.reset(new PositionGoal(link, V(p))); break;
        case BIOIK_GOAL_ORIENTATION: goal.reset(new OrientationGoal(link, q)); break;
        case BIOIK_GOAL_POSE:
        {
            auto* x = new PoseGoal(link, V(p), q);
            x->setRotationScale(p[7]);
            goal.reset(x);
            break;
        }
        case BIOIK_GOAL_LOOK_AT: goal.reset(new LookAtGoal(link, V(p), V(p + 3))); break;
        case BIOIK_GOAL_MAX_DISTANCE: goal.reset(new MaxDistanceGoal(link, V(p), p[3])); break;
        case BIOIK_GOAL_MIN_DISTANCE: goal.reset(new MinDistanceGoal(link, V(p), p[3])); break;
        case BIOIK_GOAL_LINE: goal.reset(new LineGoal(link, V(p), V(p + 3))); break;
        case BIOIK_GOAL_PLANE: goal.reset(new PlaneGoal(link, V(p), V(p + 3))); break;
        case BIOIK_GOAL_SIDE: goal.reset(new SideGoal(link, V(p), V(p + 3))); break;
        case BIOIK_GOAL_DIRECTION: goal.reset(new DirectionGoal(link, V(p), V(p + 3))); break;
        case BIOIK_GOAL_CONE: goal.reset(new ConeGoal(link, V(p), p[3], V(p + 4), V(p + 7), p[10])); break;
        case BIOIK_GOAL_AVOID_JOINT_LIMITS: goal.reset(new AvoidJointLimitsGoal(bg.weight, bg.secondary != 0)), link_goal = false; break;
        case BIOIK_GOAL_CENTER_JOINTS: goal.reset(new CenterJointsGoal(bg.weight, bg.secondary != 0)), link_goal = false; break;
        case BIOIK_GOAL_MINIMAL_DISPLACEMENT: goal.reset(new MinimalDisplacementGoal(bg.weight, bg.secondary != 0)), link_goal = false; break;
        case BIOIK_GOAL_REGULARIZATION:
            if(bg.secondary) throw std::runtime_error("ref harness: RegularizationGoal has no secondary form");
            goal.reset(new RegularizationGoal(bg.weight)), link_goal = false;
            break;
        case BIOIK_GOAL_JOINT_VARIABLE: goal.reset(new JointVariableGoal(robot.variable_names_[bg.var], p[0], bg.weight, bg.secondary != 0)), link_goal = false; break;
        case BIOIK_GOAL_BALANCE:
        {
            if(bg.secondary) throw std::runtime_error("ref harness: BalanceGoal has no secondary form");
            auto* x = new BalanceGoal(V(p), bg.weight);
            x->setAxis(V(p + 3));
            goal.reset(x), link_goal = false;
            break;
        }
        default: throw std::runtime_error("ref harness: goal type not mapped");
        }
        if(link_goal && bg.secondary) throw std::runtime_error("ref harness: link goals have no public way to become secondary");
        goal->setWeight(bg.weight);
        out.ptrs.push_back(goal.get());
        out.owned.push_back(std::move(goal));
    }
}

struct ProtoCache
{
    std::string key;
    std::shared_ptr<moveit::core::RobotModel> model;
    moveit::core::JointModelGroup group;
    IKParams params;
    std::unique_ptr<IKSolver> proto;
};
ProtoCache g_proto;

template <class T> void appendBytes(std::string& k, const T* p, size_t n)
{
    if(p) k.append((const char*)p, n * sizeof(T));
    k.push_back('|');
}

void dropProtoCache() { g_proto = ProtoCache(); }

ProtoCache& protoCache(const BioikRobot* r, const BioikProblem* problem, const char* name, uint32_t table_seed)
{
    std::string key = std::string(name) + "#" + std::to_string(table_seed) + "#";
    appendBytes(key, &r->n_links, 1), appendBytes(key, &r->n_vars, 1);
    appendBytes(key, r->link_parent, r->n_links), appendBytes(key, r->joint_type, r->n_links), appendBytes(key, r->joint_first_var, r->n_links);
    appendBytes(key, r->link_origin, 7 * (size_t)r->n_links), appendBytes(key, r->joint_axis, 3 * (size_t)r->n_links);
    appendBytes(key, r->joint_mimic, r->n_links), appendBytes(key, r->joint_mimic_factor, r->joint_mimic ? r->n_links : 0), appendBytes(key, r->joint_mimic_offset, r->joint_mimic ? r->n_links : 0);
    appendBytes(key, r->var_min, r->n_vars), appendBytes(key, r->var_max, r->n_vars), appendBytes(key, r->var_bounded, r->n_vars), appendBytes(key, r->var_max_velocity, r->n_vars);
    appendBytes(key, r->link_mass, r->link_mass ? r->n_links : 0), appendBytes(key, r->link_com, r->link_com ? 3 * (size_t)r->n_links : 0);
    appendBytes(key, problem->active_vars, problem->n_active);
    appendBytes(key, &problem->dpos, 1), appendBytes(key, &problem->drot, 1), appendBytes(key, &problem->dtwist, 1);
    if(g_proto.proto && g_proto.key == key) return g_proto;
    dropProtoCache();
    g_proto.model = makeRobot(r);
    // joint group = the joints owning the problem's active variables, in that order
    g_proto.group.parent_ = g_proto.model.get();
    for(int i = 0; i < problem->n_active; i++)
    {
        g_proto.group.variable_names_.push_back(g_proto.model->variable_names_[problem->active_vars[i]]);
        if(g_proto.group.active_joints_.empty() || g_proto.group.active_joints_.back() != g_proto.model->joint_of_variable_[problem->active_vars[i]]) // one entry per joint (a floating joint owns 7 variables)
            g_proto.group.active_joints_.push_back(g_proto.model->joint_of_variable_[problem->active_vars[i]]);
    }
    IKParams& params = g_proto.params;
    params.robot_model = g_proto.model;
    params.joint_model_group = &g_proto.group;
    params.solver_class_name = name;
    params.enable_counter = false;
    params.thread_count = 1;
    params.random_seed = (int)table_seed;
    params.dpos = problem->dpos, params.drot = problem->drot, params.dtwist = problem->dtwist;
    params.opt_no_wipeout = false, params.population_size = 8, params.elite_count = 4, params.linear_fitness = false;
    g_proto.proto.reset(IKFactory::create(name, params)); // fills the static lookup tables from table_seed
    g_proto.key = key;
    return g_proto;
}

template <class F> void parallelFor(int n, int nthreads, F f)
{
    if(nthreads <= 1 || n <= 1)
    {
        for(int i = 0; i < n; i++) f(i);
        return;
    }
    std::atomic<int> next(0);
    std::vector<std::thread> pool;
    for(int t = 0; t < nthreads; t++)
        pool.emplace_back([&]() {
            for(;;)
            {
                int i = next.fetch_add(1);
                if(i >= n) break;
                f(i);
            }
        });
    for(auto& t : pool) t.join();
}

// Quirk Q2 (forward_kinematics.h:940): computeApproximateMutation1 skips the tips a variable does not move, so the
// memetic gradient probe (ik_evolution_2.cpp:470-476) evaluates them on whatever phenotypes3[0] held before; in a fresh
// solver that is uninitialised heap memory.  Give the buffer a DEFINED initial content (identity frames) so that
// multi-tip runs are reproducible; the oracle's emulation switch (flags bit3) starts from the same content.
template <int M> void defineProbeBuffer(IKSolver* s, size_t tip_count)
{
    auto* e = dynamic_cast<IKEvolution2<M>*>(s);
    if(!e) return;
    e->phenotypes3.resize(1);
    e->phenotypes3[0].assign(tip_count, Frame::identity());
}

// The reference sizes its child pool once, in initialize(): children.resize(2 + 16) (ik_evolution_2.cpp:137-138,182);
// every loop of reproduce() / step() is then driven by children.size().  BASELINE.json's configurations use a pool
// of 128, so the harness re-sizes that (public) vector after initialize() - the reference's code is untouched and
// runs the larger population by itself.  population == 18 leaves the solver exactly as it initialised itself.
template <int M> void setPopulation(IKSolver* s, size_t population, size_t gene_count)
{
    auto* e = dynamic_cast<IKEvolution2<M>*>(s);
    if(!e || e->children.size() == population) return;
    e->children.resize(population);
    for(auto& child : e->children) child.genes.resize(gene_count), child.gradients.resize(gene_count);
}

template <int M> void traceOut(IKSolver* s, size_t n, int b, double* out_genes, double* out_gradients, double* out_species_fitness)
{
    auto* e = dynamic_cast<IKEvolution2<M>*>(s);
    if(!e) return;
    for(int sp = 0; sp < 2; sp++)
    {
        for(int k = 0; k < 2; k++)
        {
            if(out_genes) std::copy(e->species[sp].individuals[k].genes.begin(), e->species[sp].individuals[k].genes.end(), out_genes + (((size_t)b * 2 + sp) * 2 + k) * n);
            if(out_gradients) std::copy(e->species[sp].individuals[k].gradients.begin(), e->species[sp].individuals[k].gradients.end(), out_gradients + (((size_t)b * 2 + sp) * 2 + k) * n);
        }
        if(out_species_fitness) out_species_fitness[(size_t)b * 2 + sp] = e->species[sp].fitness;
    }
}
} // namespace

extern "C" {

const char* ref_last_error() { return g_error.c_str(); }

// 1: sin / cos / acos of the arithmetic contract (det_sincos, det_acos) inside the reference's code; 0: libm (default)
void ref_set_contract_math(int on)
{
    bio_ik::g_contract_math = on;
    tf2::vector3AngleAcosHook() = on ? &bioik_oracle::det_acos : nullptr;
    moveit::core::JointModel::planarSinCosHook() = on ? &bioik_oracle::det_sincos : nullptr;
}

// Same signature as oracle_solve_batch (tables argument unused: the reference owns its static tables).
int ref_solve_batch(const BioikRobot* robot, const BioikProblem* problem, const BioikSolverCfg* cfg, void*, int B, const double* goal_params, const double* seeds, const uint32_t* rng_seeds, int steps, int early_exit, int, int nthreads,
                    double* out_solutions, double* out_fitness, int32_t* out_success, int32_t* out_steps, double* out_genes, double* out_gradients, double* out_species_fitness)
{
    try
    {
        const char* name = cfg->memetic == 'q' ? "bio2_memetic" : (cfg->memetic == 'l' ? "bio2_memetic_l" : "bio2");
        if(cfg->generations != (cfg->memetic ? 8 : 16) || cfg->memetic_iters != 8 || cfg->population < 4)
            throw std::runtime_error("the reference hard-codes 8/16 generations per step and 8 memetic iterations (src/ik_evolution_2.cpp:349-350,453)");
        // One prototype solver per (robot, joint group, solver class, table seed), kept across calls like the solver a
        // plugin instance owns: constructing it fills the reference's two static 2^23-entry lookup tables (Random::Random,
        // ik_base.h:118-125), which belongs to set-up, not to the solve that bench.py times.
        ProtoCache& pc = protoCache(robot, problem, name, cfg->table_seed);
        auto& model = pc.model;
        auto& group = pc.group;
        IKParams& params = pc.params;
        auto& proto = pc.proto;
        const size_t n_vars = model->getVariableCount();
        std::atomic<int> failed(0);
        std::string err;
        parallelFor(B, nthreads, [&](int b) {
            try
            {
                GoalSet goals;
                makeGoals(*model, problem, goal_params ? goal_params + (size_t)b * problem->n_goals * BIOIK_GOAL_NPARAM : nullptr, goals);
                Problem pr;
                pr.initial_guess.assign(seeds + (size_t)b * n_vars, seeds + (size_t)(b + 1) * n_vars);
                pr.timeout = 0;
                pr.initialize(model, &group, params, goals.ptrs, nullptr);
                // the reference's own Problem::initialize must agree with the flattened problem it was given
                if(pr.active_variables.size() != (size_t)problem->n_active || pr.tip_link_indices.size() != (size_t)problem->n_tips) throw std::runtime_error("Problem::initialize disagrees with the flattened problem (sizes)");
                for(int i = 0; i < problem->n_active; i++)
                    if((int)pr.active_variables[i] != problem->active_vars[i]) throw std::runtime_error("Problem::initialize disagrees with the flattened problem (active variable order)");
                for(int i = 0; i < problem->n_tips; i++)
                    if((int)pr.tip_link_indices[i] != problem->tip_links[i]) throw std::runtime_error("Problem::initialize disagrees with the flattened problem (tip order)");
                std::unique_ptr<IKSolver> solver(IKFactory::clone(proto.get()));
                solver->rng = std::minstd_rand(rng_seeds[b]);
                solver->canceled = false;
                solver->initialize(pr);
                setPopulation<'q'>(solver.get(), cfg->population, pr.active_variables.size()), setPopulation<'l'>(solver.get(), cfg->population, pr.active_variables.size()),
                    setPopulation<0>(solver.get(), cfg->population, pr.active_variables.size());
                defineProbeBuffer<'q'>(solver.get(), pr.tip_link_indices.size()), defineProbeBuffer<'l'>(solver.get(), pr.tip_link_indices.size());
                int done = 0;
                bool success = false;
                while(done < steps)
                {
                    int burst = std::min(4, steps - done); // src/ik_parallel.h:165-168
                    for(int k = 0; k < burst; k++) solver->step();
                    done += burst;
                    std::vector<double> result = solver->getSolution();
                    solver->model.applyConfiguration(result);
                    success = solver->checkSolution(result, solver->model.getTipFrames());
                    if(success && early_exit) break;
                }
                std::vector<double> result = solver->getSolution();
                solver->model.applyConfiguration(result);
                if(out_success) out_success[b] = solver->checkSolution(result, solver->model.getTipFrames());
                if(out_fitness) out_fitness[b] = solver->computeFitness(result, solver->model.getTipFrames());
                if(out_solutions) std::copy(result.begin(), result.end(), out_solutions + (size_t)b * n_vars);
                if(out_steps) out_steps[b] = done;
                size_t n = pr.active_variables.size();
                if(cfg->memetic == 'q') traceOut<'q'>(solver.get(), n, b, out_genes, out_gradients, out_species_fitness);
                if(cfg->memetic == 'l') traceOut<'l'>(solver.get(), n, b, out_genes, out_gradients, out_species_fitness);
                if(cfg->memetic == 0) traceOut<0>(solver.get(), n, b, out_genes, out_gradients, out_species_fitness);
            }
            catch(std::exception& e)
            {
                if(!failed.exchange(1)) err = e.what();
            }
        });
        if(failed)
        {
            g_error = err;
            return 1;
        }
        return 0;
    }
    catch(std::exception& e)
    {
        g_error = e.what();
        return 1;
    }
}

// RobotFK_Fast_Base::applyConfiguration + initializeMutationApproximator + computeApproximateMutations +
// computeFitnessActiveVariables of the reference for genotypes [B][M][n] at base points [B][n_vars]
// (same contract as oracle_approx_fitness_batch); optionally the tip frames [B][T][7] and delta frames [B][T][n][7].
int ref_approx_fitness_batch(const BioikRobot* robot, const BioikProblem* problem, int B, int M, const double* goal_params, const double* seeds, const double* base_variables, const double* genotypes, double* out_primary,
                             double* out_secondary, double* out_tips, double* out_delta, double* out_frames)
{
    try
    {
        auto model = makeRobot(robot);
        moveit::core::JointModelGroup group;
        group.parent_ = model.get();
        for(int i = 0; i < problem->n_active; i++)
        {
            group.variable_names_.push_back(model->variable_names_[problem->active_vars[i]]);
            if(group.active_joints_.empty() || group.active_joints_.back() != model->joint_of_variable_[problem->active_vars[i]]) group.active_joints_.push_back(model->joint_of_variable_[problem->active_vars[i]]);
        }
        IKParams params;
        params.robot_model = model;
        params.joint_model_group = &group;
        params.solver_class_name = "bio2_memetic";
        params.enable_counter = false, params.thread_count = 1, params.random_seed = 1;
        params.dpos = problem->dpos, params.drot = problem->drot, params.dtwist = problem->dtwist;
        params.opt_no_wipeout = false, params.population_size = 8, params.elite_count = 4, params.linear_fitness = false;
        dropProtoCache(); // the constructor below refills the static lookup tables
        std::unique_ptr<IKSolver> solver(IKFactory::create("bio2_memetic", params));
        const size_t n_vars = model->getVariableCount(), n = problem->n_active, T = problem->n_tips;
        for(int b = 0; b < B; b++)
        {
            GoalSet goals;
            makeGoals(*model, problem, goal_params ? goal_params + (size_t)b * problem->n_goals * BIOIK_GOAL_NPARAM : nullptr, goals);
            Problem pr;
            pr.initial_guess.assign(seeds + (size_t)b * n_vars, seeds + (size_t)(b + 1) * n_vars);
            pr.initialize(model, &group, params, goals.ptrs, nullptr);
            solver->initialize(pr);
            std::vector<double> base(base_variables + (size_t)b * n_vars, base_variables + (size_t)(b + 1) * n_vars);
            solver->model.applyConfiguration(base);
            solver->model.initializeMutationApproximator(solver->problem.active_variables);
            if(out_tips)
                for(size_t t = 0; t < T; t++)
                {
                    const Frame& f = solver->model.getTipFrame(t);
                    double* o = out_tips + ((size_t)b * T + t) * 7;
                    o[0] = f.pos.x(), o[1] = f.pos.y(), o[2] = f.pos.z(), o[3] = f.rot.x(), o[4] = f.rot.y(), o[5] = f.rot.z(), o[6] = f.rot.w();
                }
            std::vector<const double*> gptr(M);
            for(int m = 0; m < M; m++) gptr[m] = genotypes + ((size_t)b * M + m) * n;
            std::vector<aligned_vector<Frame>> ph;
            solver->model.computeApproximateMutations(M, gptr.data(), ph);
            for(int m = 0; m < M; m++)
            {
                if(out_primary) out_primary[(size_t)b * M + m] = solver->computeFitnessActiveVariables(ph[m], gptr[m]);
                if(out_frames)
                    for(size_t t = 0; t < T; t++)
                    {
                        const Frame& f = ph[m][t];
                        double* o = out_frames + (((size_t)b * M + m) * T + t) * 7;
                        o[0] = f.pos.x(), o[1] = f.pos.y(), o[2] = f.pos.z(), o[3] = f.rot.x(), o[4] = f.rot.y(), o[5] = f.rot.z(), o[6] = f.rot.w();
                    }
                if(out_secondary) out_secondary[(size_t)b * M + m] = solver->computeSecondaryFitnessActiveVariables(gptr[m]);
            }
            if(out_delta)
            {
                // delta frames recovered exactly as differences are not available publicly: apply unit steps
                for(size_t t = 0; t < T; t++)
                    for(size_t i = 0; i < n; i++)
                    {
                        aligned_vector<Frame> in, out;
                        in.resize(T), out.resize(T);
                        for(size_t k = 0; k < T; k++) in[k] = Frame(tf2::Vector3(0, 0, 0), tf2::Quaternion(0, 0, 0, 0)), out[k] = in[k];
                        solver->model.computeApproximateMutation1(solver->problem.active_variables[i], 1.0, in, out);
                        double* o = out_delta + (((size_t)b * T + t) * n + i) * 7;
                        o[0] = out[t].pos.x(), o[1] = out[t].pos.y(), o[2] = out[t].pos.z(), o[3] = out[t].rot.x(), o[4] = out[t].rot.y(), o[5] = out[t].rot.z(), o[6] = out[t].rot.w();
                    }
            }
        }
        return 0;
    }
    catch(std::exception& e)
    {
        g_error = e.what();
        return 1;
    }
}

// The goal parameters the reference actually STORES for the given flattened records, read back through its
// public getters: several constructors normalise their argument (goal_types.h:110,139,286,314), which may move
// an already normalised vector by an ulp.  Pinning tests feed these values to the oracle so both sides compute
// on identical numbers.  gp_in / gp_out: [B][n_goals][BIOIK_GOAL_NPARAM].
int ref_effective_goal_params(const BioikRobot* robot, const BioikProblem* problem, int B, const double* gp_in, double* gp_out)
{
    try
    {
        auto model = makeRobot(robot);
        auto W3 = [](double* o, const tf2::Vector3& v) { o[0] = v.x(), o[1] = v.y(), o[2] = v.z(); };
        auto W4 = [](double* o, const tf2::Quaternion& q) { o[0] = q.x(), o[1] = q.y(), o[2] = q.z(), o[3] = q.w(); };
        for(int b = 0; b < B; b++)
        {
            GoalSet goals;
            makeGoals(*model, problem, gp_in + (size_t)b * problem->n_goals * BIOIK_GOAL_NPARAM, goals);
            for(int g = 0; g < problem->n_goals; g++)
            {
                const double* in = gp_in + ((size_t)b * problem->n_goals + g) * BIOIK_GOAL_NPARAM;
                double* o = gp_out + ((size_t)b * problem->n_goals + g) * BIOIK_GOAL_NPARAM;
                std::copy(in, in + BIOIK_GOAL_NPARAM, o);
                const Goal* goal = goals.ptrs[g];
                if(auto* x = dynamic_cast<const PositionGoal*>(goal)) W3(o, x->getPosition());
                if(auto* x = dynamic_cast<const OrientationGoal*>(goal)) W4(o + 3, x->getOrientation());
                if(auto* x = dynamic_cast<const PoseGoal*>(goal)) W3(o, x->getPosition()), W4(o + 3, x->getOrientation()), o[7] = x->getRotationScale();
                if(auto* x = dynamic_cast<const LookAtGoal*>(goal)) W3(o, x->getAxis()), W3(o + 3, x->getTarget());
                if(auto* x = dynamic_cast<const MaxDistanceGoal*>(goal)) W3(o, x->getTarget()), o[3] = x->getDistance();
                if(auto* x = dynamic_cast<const MinDistanceGoal*>(goal)) W3(o, x->getTarget()), o[3] = x->getDistance();
                if(auto* x = dynamic_cast<const LineGoal*>(goal)) W3(o, x->getPosition()), W3(o + 3, x->getDirection());
                if(auto* x = dynamic_cast<const PlaneGoal*>(goal)) W3(o, x->getPosition()), W3(o + 3, x->getNormal());
                if(auto* x = dynamic_cast<const SideGoal*>(goal)) W3(o, x->getAxis()), W3(o + 3, x->getDirection());
                if(auto* x = dynamic_cast<const DirectionGoal*>(goal)) W3(o, x->getAxis()), W3(o + 3, x->getDirection());
                if(auto* x = dynamic_cast<const ConeGoal*>(goal)) W3(o, x->getPosition()), o[3] = x->getPositionWeight(), W3(o + 4, x->getAxis()), W3(o + 7, x->getDirection()), o[10] = x->getAngle();
                if(auto* x = dynamic_cast<const JointVariableGoal*>(goal)) o[0] = x->getVariablePosition();
                if(auto* x = dynamic_cast<const BalanceGoal*>(goal)) W3(o, x->getTarget()), W3(o + 3, x->getAxis());
            }
        }
        return 0;
    }
    catch(std::exception& e)
    {
        g_error = e.what();
        return 1;
    }
}

// The link origin frames the reference actually computes with: RobotJointEvaluator builds them with
// Frame(link_model->getJointOriginTransform()) (forward_kinematics.h:203), i.e. an Isometry3d -> quaternion
// conversion of what the C ABI hands over as a quaternion.  A quaternion -> matrix -> quaternion round trip may
// move the last bit, so the pinning tests give the oracle exactly these frames.  out: [n_links][7].
int ref_effective_link_origins(const BioikRobot* robot, double* out)
{
    try
    {
        auto model = makeRobot(robot);
        for(int l = 0; l < robot->n_links; l++)
        {
            Frame f(model->links_[l]->getJointOriginTransform());
            double* o = out + 7 * l;
            o[0] = f.pos.x(), o[1] = f.pos.y(), o[2] = f.pos.z(), o[3] = f.rot.x(), o[4] = f.rot.y(), o[5] = f.rot.z(), o[6] = f.rot.w();
        }
        return 0;
    }
    catch(std::exception& e)
    {
        g_error = e.what();
        return 1;
    }
}

// the lookup tables the reference filled (for a direct comparison with Tables / make_tables)
const double* ref_table(int which, uint32_t seed)
{
    static std::unique_ptr<Random> r;
    dropProtoCache();
    r.reset(new Random(seed));
    return which ? r->random_gauss_buffer : r->random_buffer;
}
}
