// ik_evolution_2_b200.cpp — the ONE translation unit a bio_ik maintainer adds to the reference tree (next to
// src/ik_evolution_2.cpp, linked with -lbioik_b200) to run the bio2 family on an H100 behind the reference's own solver seam.
//
// It registers three IKBase subclasses with IKFactory, exactly like src/ik_evolution_2.cpp:652-654 registers the CPU ones:
//     mode: bio2_b200 | bio2_memetic_b200 | bio2_memetic_l_b200        (ROS parameter read at src/kinematics_plugin.cpp:252-253)
// MoveIt keeps loading bio_ik/BioIKKinematicsPlugin; the plugin, IKParallel, RobotInfo / Problem construction and goal parsing
// stay as they are.  The class implements the four virtuals IKParallel::solverthread uses (src/ik_parallel.h:156,165-181):
//     initialize(problem)  -> bioik_set_problem (when the problem STRUCTURE changed) + bioik_begin (this query's numbers)
//     step()               -> bioik_step(ctx, 1): one IKEvolution2::step of every island, state resident on the device
//     getSolution()        -> bioik_get_solution: the best island, chosen the way IKParallel::solve chooses among its threads
//     concurrency()        -> 1: one host thread drives the GPU (src/ik_base.h:209)
// One solver object = `islands` differently seeded device runs of the query (BIOIK_B200_ISLANDS, default 64), where the
// reference's thread pool runs bit-identical clones (src/ik_parallel.h:119-127).  With params.thread_count > 1 IKParallel
// copy-constructs the solver through IKFactory::clone (src/utils.h:423): every copy owns a device context of its own and
// seeds its islands from its thread_index.
//
// Only public interfaces of the reference are used (IKBase, Problem::GoalInfo, the goal classes' getters, moveit::core::RobotModel).
// Goals without a closed form on the device (TouchGoal, JointFunctionGoal, LinkFunctionGoal) raise the reference's ERROR():
// keep mode=bio2_memetic for those queries.
#include "ik_base.h"

#include <bio_ik/goal_types.h>

#include <bioik_b200.h>

#include <cstdlib>
#include <cstring>

namespace bio_ik
{

template <int memetic> struct IKEvolution2B200 : IKBase
{
    // the flattened moveit::core::RobotModel (SURVEY.md Appendix B), kept for re-creating the context in copies
    struct RobotTable
    {
        std::vector<int32_t> parent, jtype, first_var, mimic, bounded;
        std::vector<double> origin, axis, mfac, moff, vmin, vmax, vvel, mass, com;
    };
    RobotTable table;
    bioik_ctx* ctx = nullptr;
    int islands = 64, device = 0, stream_stride = 0;

    // what bioik_set_problem was last called with: a new query with the same structure only needs bioik_begin
    std::vector<int32_t> set_tips, set_active;
    std::vector<BioikGoal> set_goals;

    mutable std::vector<double> solution;
    mutable bool solution_current = false;
    mutable double solution_fitness = 0;
    mutable int32_t solution_success = 0, solution_island = 0, solution_steps = 0;

    static int envInt(const char* name, int fallback)
    {
        const char* v = getenv(name);
        return v && atoi(v) > 0 ? atoi(v) : fallback;
    }

    void flattenRobot(const moveit::core::RobotModel& m)
    {
        using moveit::core::JointModel;
        for(auto* link : m.getLinkModels())
        {
            auto* joint = link->getParentJointModel();
            table.parent.push_back(link->getParentLinkModel() ? (int32_t)link->getParentLinkModel()->getLinkIndex() : -1);
            int32_t t = BIOIK_JOINT_FIXED;
            switch(joint->getType())
            {
            case JointModel::REVOLUTE: t = BIOIK_JOINT_REVOLUTE; break;
            case JointModel::PRISMATIC: t = BIOIK_JOINT_PRISMATIC; break;
            case JointModel::FLOATING: t = BIOIK_JOINT_FLOATING; break;
            case JointModel::PLANAR: t = BIOIK_JOINT_PLANAR; break;
            case JointModel::FIXED: t = BIOIK_JOINT_FIXED; break;
            default: ERROR("joint type has no device implementation", joint->getName());
            }
            table.jtype.push_back(t);
            table.first_var.push_back(joint->getVariableCount() ? (int32_t)joint->getFirstVariableIndex() : -1);
            Frame f(link->getJointOriginTransform()); // the conversion RobotJointEvaluator does, src/forward_kinematics.h:203
            for(double v : {f.pos.x(), f.pos.y(), f.pos.z(), f.rot.x(), f.rot.y(), f.rot.z(), f.rot.w()}) table.origin.push_back(v);
            double ax = 0, ay = 0, az = 0; // src/forward_kinematics.h:205-212
            if(auto* j = dynamic_cast<const moveit::core::RevoluteJointModel*>(joint)) ax = j->getAxis().x(), ay = j->getAxis().y(), az = j->getAxis().z();
            if(auto* j = dynamic_cast<const moveit::core::PrismaticJointModel*>(joint)) ax = j->getAxis().x(), ay = j->getAxis().y(), az = j->getAxis().z();
            table.axis.insert(table.axis.end(), {ax, ay, az});
            table.mimic.push_back(joint->getMimic() ? (int32_t)joint->getMimic()->getChildLinkModel()->getLinkIndex() : -1);
            table.mfac.push_back(joint->getMimicFactor());
            table.moff.push_back(joint->getMimicOffset());
            // URDF inertial, as BalanceGoal::describe reads it (src/goal_types.cpp:236-250)
            double mass = 0, cx = 0, cy = 0, cz = 0;
            if(m.getURDF())
                if(auto link_urdf = m.getURDF()->getLink(link->getName()))
                    if(link_urdf->inertial) mass = link_urdf->inertial->mass, cx = link_urdf->inertial->origin.position.x, cy = link_urdf->inertial->origin.position.y, cz = link_urdf->inertial->origin.position.z;
            table.mass.push_back(mass);
            table.com.insert(table.com.end(), {cx, cy, cz});
        }
        for(auto& name : m.getVariableNames())
        {
            auto& b = m.getVariableBounds(name); // what RobotInfo reads, include/bio_ik/robot_info.h:73-105
            table.vmin.push_back(b.min_position_);
            table.vmax.push_back(b.max_position_);
            table.bounded.push_back(b.position_bounded_ ? 1 : 0);
            table.vvel.push_back(b.max_velocity_);
        }
    }

    void createContext()
    {
        BioikRobot r;
        memset(&r, 0, sizeof(r));
        r.n_links = (int32_t)table.parent.size(), r.n_vars = (int32_t)table.vmin.size();
        r.link_parent = table.parent.data(), r.joint_type = table.jtype.data(), r.joint_first_var = table.first_var.data();
        r.link_origin = table.origin.data(), r.joint_axis = table.axis.data();
        r.joint_mimic = table.mimic.data(), r.joint_mimic_factor = table.mfac.data(), r.joint_mimic_offset = table.moff.data();
        r.var_min = table.vmin.data(), r.var_max = table.vmax.data(), r.var_bounded = table.bounded.data(), r.var_max_velocity = table.vvel.data();
        r.link_mass = table.mass.data(), r.link_com = table.com.data();
        // the constants src/ik_evolution_2.cpp hard-codes: 2 + 16 children (:137-138,182), 8 generations per step (16 without the
        // memetic stage, :349-351), 8 line-search iterations (:453); the lookup tables are seeded like Random(p.random_seed)
        BioikSolverCfg cfg;
        cfg.population = 18, cfg.generations = memetic ? 8 : 16, cfg.memetic = memetic, cfg.memetic_iters = 8;
        cfg.table_seed = (uint32_t)params.random_seed, cfg.device = device;
        ctx = nullptr;
        if(bioik_create(&r, &cfg, &ctx) != BIOIK_OK) ERROR("bioik_create", bioik_last_error(nullptr));
        // 0 (default): the islands are clones of one random stream like IKParallel's threads; k > 0: island i starts i * k steps into it
        if(stream_stride > 0 && bioik_set_option(ctx, BIOIK_OPT_ISLAND_STREAM_STRIDE, stream_stride) != BIOIK_OK) ERROR("bioik_set_option", bioik_last_error(ctx));
        set_tips.clear(), set_active.clear(), set_goals.clear();
    }

    IKEvolution2B200(const IKParams& p)
        : IKBase(p)
    {
        islands = envInt("BIOIK_B200_ISLANDS", 64);
        device = envInt("BIOIK_B200_DEVICE", 0);
        stream_stride = envInt("BIOIK_B200_ISLAND_STREAM_STRIDE", 0);
        flattenRobot(*p.robot_model);
        createContext();
    }
    // IKFactory::clone copy-constructs (src/utils.h:423): the copy gets a device context of its own
    IKEvolution2B200(const IKEvolution2B200& o)
        : IKBase(o)
        , table(o.table)
        , islands(o.islands)
        , device(o.device)
        , stream_stride(o.stream_stride)
    {
        createContext();
    }
    IKEvolution2B200& operator=(const IKEvolution2B200&) = delete;
    ~IKEvolution2B200() { bioik_destroy(ctx); }

    static void put3(double* o, const tf2::Vector3& v) { o[0] = v.x(), o[1] = v.y(), o[2] = v.z(); }
    static void put4(double* o, const tf2::Quaternion& q) { o[0] = q.x(), o[1] = q.y(), o[2] = q.z(), o[3] = q.w(); }

    // Problem::GoalInfo -> BioikGoal: one branch per closed-form goal class of include/bio_ik/goal_types.h (p[] layouts: bioik_b200.h)
    BioikGoal flattenGoal(const Problem::GoalInfo& gi, bool secondary) const
    {
        BioikGoal g;
        memset(&g, 0, sizeof(g));
        g.tip = (int32_t)gi.tip_index;
        g.secondary = secondary ? 1 : 0;
        g.weight = gi.weight;
        double* p = g.p;
        const Goal* goal = gi.goal;
        if(auto* x = dynamic_cast<const PoseGoal*>(goal))
            g.type = BIOIK_GOAL_POSE, put3(p, x->getPosition()), put4(p + 3, x->getOrientation()), p[7] = x->getRotationScale();
        else if(auto* x = dynamic_cast<const PositionGoal*>(goal))
            g.type = BIOIK_GOAL_POSITION, put3(p, x->getPosition());
        else if(auto* x = dynamic_cast<const OrientationGoal*>(goal))
            g.type = BIOIK_GOAL_ORIENTATION, put4(p + 3, x->getOrientation());
        else if(auto* x = dynamic_cast<const LookAtGoal*>(goal))
            g.type = BIOIK_GOAL_LOOK_AT, put3(p, x->getAxis()), put3(p + 3, x->getTarget());
        else if(auto* x = dynamic_cast<const MaxDistanceGoal*>(goal))
            g.type = BIOIK_GOAL_MAX_DISTANCE, put3(p, x->getTarget()), p[3] = x->getDistance();
        else if(auto* x = dynamic_cast<const MinDistanceGoal*>(goal))
            g.type = BIOIK_GOAL_MIN_DISTANCE, put3(p, x->getTarget()), p[3] = x->getDistance();
        else if(auto* x = dynamic_cast<const LineGoal*>(goal))
            g.type = BIOIK_GOAL_LINE, put3(p, x->getPosition()), put3(p + 3, x->getDirection());
        else if(auto* x = dynamic_cast<const PlaneGoal*>(goal))
            g.type = BIOIK_GOAL_PLANE, put3(p, x->getPosition()), put3(p + 3, x->getNormal());
        else if(auto* x = dynamic_cast<const SideGoal*>(goal))
            g.type = BIOIK_GOAL_SIDE, put3(p, x->getAxis()), put3(p + 3, x->getDirection());
        else if(auto* x = dynamic_cast<const DirectionGoal*>(goal))
            g.type = BIOIK_GOAL_DIRECTION, put3(p, x->getAxis()), put3(p + 3, x->getDirection());
        else if(auto* x = dynamic_cast<const ConeGoal*>(goal))
            g.type = BIOIK_GOAL_CONE, put3(p, x->getPosition()), p[3] = x->getPositionWeight(), put3(p + 4, x->getAxis()), put3(p + 7, x->getDirection()), p[10] = x->getAngle();
        else if(dynamic_cast<const AvoidJointLimitsGoal*>(goal))
            g.type = BIOIK_GOAL_AVOID_JOINT_LIMITS;
        else if(dynamic_cast<const CenterJointsGoal*>(goal))
            g.type = BIOIK_GOAL_CENTER_JOINTS;
        else if(dynamic_cast<const RegularizationGoal*>(goal))
            g.type = BIOIK_GOAL_REGULARIZATION;
        else if(dynamic_cast<const MinimalDisplacementGoal*>(goal))
            g.type = BIOIK_GOAL_MINIMAL_DISPLACEMENT;
        else if(auto* x = dynamic_cast<const JointVariableGoal*>(goal))
            g.type = BIOIK_GOAL_JOINT_VARIABLE, g.var = (int32_t)params.robot_model->getVariableIndex(x->getVariableName()), p[0] = x->getVariablePosition();
        else if(auto* x = dynamic_cast<const BalanceGoal*>(goal))
            g.type = BIOIK_GOAL_BALANCE, put3(p, x->getTarget()), put3(p + 3, x->getAxis()); // its links: every link with mass, already tips of the problem
        else
            ERROR("goal class has no device implementation: keep a CPU solver mode for this query"); // Touch, JointFunction, LinkFunction
        return g;
    }

    static bool sameStructure(const BioikGoal& a, const BioikGoal& b) { return a.type == b.type && a.tip == b.tip && a.secondary == b.secondary && a.var == b.var && a.weight == b.weight; }

    void initialize(const Problem& problem) override
    {
        IKBase::initialize(problem); // keeps `model` usable for the driver's own exact FK + checkSolution (src/ik_parallel.h:175-181)
        std::vector<BioikGoal> goals;
        for(auto& g : this->problem.goals) goals.push_back(flattenGoal(g, false));
        for(auto& g : this->problem.secondary_goals) goals.push_back(flattenGoal(g, true));
        std::vector<int32_t> tips(this->problem.tip_link_indices.begin(), this->problem.tip_link_indices.end());
        std::vector<int32_t> active(this->problem.active_variables.begin(), this->problem.active_variables.end());
        bool same = tips == set_tips && active == set_active && goals.size() == set_goals.size();
        for(size_t i = 0; same && i < goals.size(); i++) same = sameStructure(goals[i], set_goals[i]);
        if(!same)
        {
            BioikProblem bp;
            memset(&bp, 0, sizeof(bp));
            bp.n_tips = (int32_t)tips.size(), bp.tip_links = tips.data();
            bp.n_active = (int32_t)active.size(), bp.active_vars = active.data();
            bp.n_goals = (int32_t)goals.size(), bp.goals = goals.data();
            bp.dpos = params.dpos, bp.drot = params.drot, bp.dtwist = params.dtwist; // normalised like src/problem.cpp:90-95 inside the library
            if(bioik_set_problem(ctx, &bp) != BIOIK_OK) ERROR("bioik_set_problem", bioik_last_error(ctx));
            set_tips = tips, set_active = active, set_goals = goals;
        }
        // this query: goal numbers, seed, one RNG seed per island
        std::vector<double> gp(goals.size() * BIOIK_GOAL_NPARAM);
        for(size_t i = 0; i < goals.size(); i++) memcpy(&gp[i * BIOIK_GOAL_NPARAM], goals[i].p, sizeof(goals[i].p));
        std::vector<uint32_t> rs(islands);
        for(int i = 0; i < islands; i++) rs[i] = (uint32_t)params.random_seed + (uint32_t)(thread_index * islands + i);
        // early_exit 2 = the driver's `finished` flag among the islands (src/ik_parallel.h:160-186); no step budget: IKParallel's
        // timeout decides (src/ik_parallel.h:162)
        if(bioik_begin(ctx, 1, islands, gp.data(), this->problem.initial_guess.data(), rs.data(), 0, 2) != BIOIK_OK) ERROR("bioik_begin", bioik_last_error(ctx));
        solution = this->problem.initial_guess;
        solution_current = false;
    }

    void step() override
    {
        if(canceled) return; // src/ik_evolution_2.cpp:355
        if(bioik_step(ctx, 1, nullptr) != BIOIK_OK) ERROR("bioik_step", bioik_last_error(ctx));
        solution_current = false;
    }

    const std::vector<double>& getSolution() const override
    {
        if(!solution_current)
        {
            solution.resize(problem.initial_guess.size());
            // wrap = 0: the plugin wraps the angles itself (src/kinematics_plugin.cpp:580-611)
            if(bioik_get_solution(ctx, 0, solution.data(), &solution_fitness, &solution_success, &solution_island, &solution_steps) != BIOIK_OK) ERROR("bioik_get_solution", bioik_last_error(ctx));
            solution_current = true;
        }
        return solution;
    }

    size_t concurrency() const override { return 1; }
};

static IKFactory::Class<IKEvolution2B200<0>> bio2_b200("bio2_b200");
static IKFactory::Class<IKEvolution2B200<'q'>> bio2_memetic_b200("bio2_memetic_b200");
static IKFactory::Class<IKEvolution2B200<'l'>> bio2_memetic_l_b200("bio2_memetic_l_b200");
}
