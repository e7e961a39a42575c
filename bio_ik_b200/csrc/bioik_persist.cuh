// bioik_persist.cuh — the persistent solve kernel: ONE launch runs steps [s0, s1) of every run of a batch.
//
// The stepped path launches k_evolve_fast + k_serial once per step().  That costs the tail of every generation launch
// (a fractional number of waves of blocks), leaves most of the chip idle while the latency-bound serial
// kernel runs (one warp per scheduler), and round-trips through ~50 launches per solve.  Here the same two bodies
// (evolve_fast_task, serial_tasks: identical arithmetic, identical results) are work ITEMS that resident warps take from
// two queues in device memory:
//     evolve item (query q, step s)     one warp: the generations of both species of q           (src/ik_evolution_2.cpp:351-432)
//     serial item (group g, step s)     one warp, one thread per task of the group's 16 queries: memetic line search,
//                                       species block, exact FK + Jacobian + delta frames of the next step (:436-646,:341-346)
// with the dependencies of step():  evolve(q, s) x 16 -> serial(g, s) -> evolve(q, s + 1) x 16.  Groups drift apart in step
// number, so the serial item of one group runs in the shadow of the generation work of the others, and there is no
// per-step barrier whose tail every query would pay.  The state stays in HBM/L2 between items (1.7 KB per task), so any
// warp of any SM can take any item: the queues are global.
//
// Queue protocol (no blocking tickets, hence no deadlock by construction):
//   push:  i = atomicAdd(tail, k); slots[i .. i + k) = items (st.release after a __threadfence of every lane)
//   pop:   if(head < tail) ticket = atomicAdd(head, 1); then the warp watches slots[ticket] (ld.acquire) while it keeps
//          serving its other queue - a ticket beyond the tail is served by a later push, holding one never blocks
//   a warp that finds nothing sleeps 0.1 - 1.5 us and looks again; all warps leave when every group has finished step s1 - 1.
// Warp 0 of every block owns the block's serial shared-memory region and is the only one that takes serial items (it
// prefers them); every warp takes evolve items.
#pragma once

#include "bioik_evolve_fast.cuh"
#include "bioik_serial.cuh"

namespace bioik
{

constexpr int PERSIST_GROUP_QUERIES = 16; // queries per serial item = 32 tasks = one warp, one thread per task
constexpr int PERSIST_WARPS = 4;          // warps per block
// A warp that finds no work for this many polls in a row (~0.2 us each: several seconds, orders of magnitude beyond the longest
// item) raises ctr[5] and every warp leaves: a broken dependency chain must end in an error, not in a hung device.
constexpr int PERSIST_WATCHDOG_POLLS = 1 << 23;
// queue counters, 32 ints (one 128-byte line) apart: the head of the evolve queue takes one atomic per item
constexpr int PQ_HEAD_E = 0, PQ_TAIL_E = 32, PQ_HEAD_S = 64, PQ_TAIL_S = 96, PQ_DONE = 128, PQ_ABORT = 160, PQ_STATS = 192 /* 8 x u64, BIOIK_PERSIST_STATS builds */, PQ_INTS = 256;

struct PersistArgs
{
    int32_t s0, s1;    // steps [s0, s1)
    int32_t last;      // s1 is the end of the solve: the approximator of step s1 is not prepared
    int32_t prepared;  // the approximator of step s0 is already in the state (else every group starts with a PREPARE item)
    int32_t groups;    // ceil(B / PERSIST_GROUP_QUERIES)
    int32_t sm_count;  // blocks b, b + sm_count, ... tend to share an SM: their serial warps are spread over the four schedulers
    int32_t cap_e, cap_s; // slots of the two queues
    unsigned long long* slots_e; // evolve items:  (step + 1) << 32 | query
    unsigned long long* slots_s; // serial items:  phases << 56 | (step + 1) << 32 | group
    int32_t* ctr;      // [PQ_INTS] queue heads / tails, groups finished, watchdog flag (PQ_* below)
    int32_t* gcount;   // [groups] evolve items of the group's current step that have finished
};

__host__ __device__ inline unsigned long long persist_evolve_item(int step, int q) { return ((unsigned long long)(step + 1) << 32) | (unsigned)q; }
__host__ __device__ inline unsigned long long persist_serial_item(int step, int g, int phases) { return ((unsigned long long)phases << 56) | ((unsigned long long)(step + 1) << 32) | (unsigned)g; }

#ifndef BIOIK_HOSTSIM
__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long* p)
{
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u64(unsigned long long* p, unsigned long long v) { asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ int ld_relaxed_s32(const int32_t* p)
{
    int v;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void persist_sleep(int idle) { __nanosleep(idle < 4 ? 100u : (idle < 64 ? 400u : 1500u)); }
#else
static inline unsigned long long ld_acquire_u64(const unsigned long long* p) { return *(volatile const unsigned long long*)p; }
static inline void st_release_u64(unsigned long long* p, unsigned long long v) { *(volatile unsigned long long*)p = v; }
static inline int ld_relaxed_s32(const int32_t* p) { return *(volatile const int32_t*)p; }
static inline void persist_sleep(int) {}
#endif

// initial queue content of one launch: PREPARE items of every group, or - approximator already there - the evolve items of step s0
__global__ void k_persist_init(PersistArgs A, int B)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i < A.cap_e) A.slots_e[i] = (A.prepared && i < B) ? persist_evolve_item(A.s0, i) : 0ull;
    if(i < A.cap_s) A.slots_s[i] = (!A.prepared && i < A.groups) ? persist_serial_item(A.s0, i, PH_PREPARE) : 0ull;
    if(i < A.groups) A.gcount[i] = 0;
    if(i < PQ_INTS && i != PQ_STATS && (i < PQ_STATS || i >= PQ_STATS + 16))
    {
        int v = 0;
        if(i == PQ_TAIL_E) v = A.prepared ? B : 0;
        if(i == PQ_TAIL_S) v = A.prepared ? 0 : A.groups;
        if(i == PQ_DONE) v = A.s1 > A.s0 ? 0 : A.groups;
        A.ctr[i] = v;
    }
}

// One lane's view of one queue.  A warp takes a TICKET (atomicAdd on the head: always succeeds, unlike a compare-and-swap,
// which under thousands of contenders lets one through per round trip) only when the queue looks non-empty, and then
// watches ITS slot.  Several warps may see the same last item, so a ticket can lie beyond the tail: it is simply served by
// a later push.  Holding a ticket never blocks: the warp keeps looking at its other queue in the meantime.
struct PersistTicket
{
    int pending = -1;
    __device__ __forceinline__ unsigned long long poll(int32_t* head, const int32_t* tail, const unsigned long long* slots, int cap)
    {
        if(pending < 0 && ld_relaxed_s32(head) < ld_relaxed_s32(tail)) pending = atomicAdd(head, 1);
        if(pending < 0 || pending >= cap) return 0ull;
        const unsigned long long v = ld_acquire_u64(slots + pending);
        if(v != 0ull) pending = -1;
        return v;
    }
};

// T .. LPT: the generation kernel's parameters (bioik_evolve_fast.cuh); DS / FS: delta frames / link frames of the serial
// body in shared memory (bioik_serial.cuh).  Shared memory of a block: PERSIST_WARPS x (32 / LPT) evolve blocks, then one
// serial region (32 columns).
template <int T, int CH, int GSPEC, bool JOINT, int NG, bool TM, int LPT, bool DS, bool FS>
__global__ void __launch_bounds__(32 * PERSIST_WARPS, 4) k_persist(BIOIK_PROBLEM_PARAM, const DProblem* __restrict__ Pp, DState S, PersistArgs A, const double* __restrict__ mtab)
{
    extern __shared__ double smem[];
    constexpr int TPW = 32 / LPT; // tasks per warp = species of TPW / 2 queries
    static_assert(TPW == 2, "an evolve item is one query = the two species of a warp's lane groups");
    const int warp = threadIdx.x >> 5, wl = threadIdx.x & 31;
    const int lane = wl % LPT, grp = wl / LPT, lane0 = grp * LPT;
    const unsigned gmask = ((1u << LPT) - 1u) << lane0;
    const DProblem& Pg = *Pp; // the generation body indexes the problem per lane: global memory, not the constant bank
    const int n = NG ? NG : Pg.n;
    FastSmem L{n, TM ? Pg.T : T, Pg.G, JOINT ? Pg.n_joint_goals : 0, Pg.has_secondary ? 0 : 1};
    double* ev = smem + (size_t)(warp * TPW + grp) * L.total();
    double* ser = smem + (size_t)PERSIST_WARPS * TPW * L.total();
    const bool serial_warp = warp == (int)((blockIdx.x / (unsigned)max(A.sm_count, 1)) % PERSIST_WARPS) || blockDim.x < 32 * PERSIST_WARPS;

    PersistTicket ticket_e, ticket_s; // lane 0's
    int idle = 0;
#ifdef BIOIK_PERSIST_STATS
    long long t_evolve = 0, t_serial = 0, t_idle = 0, n_evolve = 0, n_serial = 0, n_polls = 0;
    const long long t_begin = clock64();
#endif
    for(;;)
    {
#ifdef BIOIK_PERSIST_STATS
        const long long t0 = clock64();
#endif
        unsigned long long item = 0ull;
        int kind = -1; // 0 evolve, 1 serial, 2 leave
        if(wl == 0)
        {
            if(serial_warp && (item = ticket_s.poll(A.ctr + PQ_HEAD_S, A.ctr + PQ_TAIL_S, A.slots_s, A.cap_s)) != 0ull)
                kind = 1;
            else if((item = ticket_e.poll(A.ctr + PQ_HEAD_E, A.ctr + PQ_TAIL_E, A.slots_e, A.cap_e)) != 0ull)
                kind = 0;
            else if((idle & 7) == 7 && (ld_relaxed_s32(A.ctr + PQ_DONE) >= A.groups || ld_relaxed_s32(A.ctr + PQ_ABORT) != 0))
                kind = 2;
            if(kind < 0 && ++idle > PERSIST_WATCHDOG_POLLS)
            {
                atomicExch(A.ctr + PQ_ABORT, 1);
                kind = 2;
            }
        }
        kind = __shfl_sync(0xffffffffu, kind, 0);
        if(kind == 2) break;
        if(kind < 0)
        {
            persist_sleep(idle);
#ifdef BIOIK_PERSIST_STATS
            t_idle += clock64() - t0, n_polls++;
#endif
            continue;
        }
        idle = 0;
        item = __shfl_sync(0xffffffffu, item, 0);
        __threadfence(); // acquire side: what the producers of this item wrote is visible to every lane from here on
        const int step = (int)((item >> 32) & 0xFFFFFFu) - 1;
        if(kind == 0)
        {
            const int q = (int)(item & 0xFFFFFFFFu);
            evolve_fast_task<T, CH, GSPEC, JOINT, NG, TM, LPT>(Pg, S, step, mtab, ev, 2 * q + grp, lane, lane0, gmask);
            __threadfence(); // release side: this lane's state writes before the completion count
            __syncwarp();
            if(wl == 0)
            {
                const int g = q / PERSIST_GROUP_QUERIES;
                const int size = min(PERSIST_GROUP_QUERIES, S.B - g * PERSIST_GROUP_QUERIES);
                if(atomicAdd(A.gcount + g, 1) == size - 1)
                {
                    // the last query of the group: hand the group to a serial warp
                    A.gcount[g] = 0;
                    __threadfence();
                    const bool prep = !(A.last && step + 1 == A.s1);
                    const int phases = (S.memetic ? PH_MEMETIC : 0) | PH_SPECIES | (prep ? PH_PREPARE : 0);
                    const int i = atomicAdd(A.ctr + PQ_TAIL_S, 1);
                    st_release_u64(A.slots_s + i, persist_serial_item(step, g, phases));
                }
            }
#ifdef BIOIK_PERSIST_STATS
            t_evolve += clock64() - t0, n_evolve++;
#endif
        }
        else
        {
            const int g = (int)(item & 0xFFFFFFFFu), phases = (int)(item >> 56);
#ifndef BIOIK_X_NOSERIAL // timing experiment only (wrong results): serial items do nothing but release the next evolve items
            serial_tasks<32, DS, FS>(P, S, step, phases, ser, wl, 2 * PERSIST_GROUP_QUERIES * g + wl);
#endif
            __threadfence();
            __syncwarp();
            const int next = phases == PH_PREPARE ? step : step + 1; // a PREPARE item opens its own step
            const int q0 = g * PERSIST_GROUP_QUERIES, size = min(PERSIST_GROUP_QUERIES, S.B - q0);
            if(next < A.s1)
            {
                int base = 0;
                if(wl == 0) base = atomicAdd(A.ctr + PQ_TAIL_E, size);
                base = __shfl_sync(0xffffffffu, base, 0);
                if(wl < size) st_release_u64(A.slots_e + base + wl, persist_evolve_item(next, q0 + wl));
            }
            else if(wl == 0)
                atomicAdd(A.ctr + PQ_DONE, 1);
#ifdef BIOIK_PERSIST_STATS
            t_serial += clock64() - t0, n_serial++;
#endif
        }
    }
#ifdef BIOIK_PERSIST_STATS
    if(wl == 0)
    {
        unsigned long long* st = (unsigned long long*)(A.ctr + PQ_STATS);
        atomicAdd(st + 0, (unsigned long long)t_evolve), atomicAdd(st + 1, (unsigned long long)t_serial), atomicAdd(st + 2, (unsigned long long)t_idle);
        atomicAdd(st + 3, (unsigned long long)n_evolve), atomicAdd(st + 4, (unsigned long long)n_serial), atomicAdd(st + 5, (unsigned long long)n_polls);
        atomicAdd(st + 6, (unsigned long long)(clock64() - t_begin)), atomicAdd(st + 7, 1ull);
    }
#endif
}

#ifdef BIOIK_HOSTSIM
typedef void (*PersistKernel)(const DProblem&, const DProblem*, DState, PersistArgs, const double*);
#else
typedef void (*PersistKernel)(const DProblem, const DProblem*, DState, PersistArgs, const double*);
#endif

// shared memory of one block of the persistent kernel for problem P (bytes); *ser_doubles = offset of the serial region
inline size_t persist_smem_bytes(const DProblem& P, int lpt, bool delta_smem, bool frames_smem)
{
    FastSmem L = fast_smem_layout(P);
    const size_t ev = (size_t)PERSIST_WARPS * (32 / lpt) * L.total();
    const size_t ser = (size_t)(serial_fixed_doubles(P) + (delta_smem ? 7 * P.T * P.n : 0) + (frames_smem ? 7 * P.L : 0)) * 32;
    return (ev + ser) * sizeof(double);
}

// The persistent kernel exists for the shapes whose whole step fits the two bodies above: the single-pose problem with 6 or 7
// genes (generation kernel with 16-lane groups, memetic step inside the serial body).  nullptr: use the stepped launches.
inline PersistKernel select_persist(const DProblem& P, int C, bool* delta_smem, bool* frames_smem)
{
    const bool single_pose = (P.G == 1 && P.goals[0].type == G_POSE && !P.goals[0].secondary && P.T == 1);
    if(!single_pose || !has_unrolled_memetic(P) || P.n_quat > 0 || C > 32 * FAST_MAX_CPL) return nullptr;
    *delta_smem = true, *frames_smem = false;
#ifdef BIOIK_SLIM
    return BIOIK_NAMED_AS(PersistKernel, k_persist<1, 4, 1, false, 7, false, 16, true, false>);
#else
    if(mtab_row(C) == 32) // population <= 34 (the reference's 18): register blocks of 2
        return P.n == 7 ? BIOIK_NAMED_AS(PersistKernel, k_persist<1, 2, 1, false, 7, false, 16, true, false>) : BIOIK_NAMED_AS(PersistKernel, k_persist<1, 2, 1, false, 6, false, 16, true, false>);
    return P.n == 7 ? BIOIK_NAMED_AS(PersistKernel, k_persist<1, 4, 1, false, 7, false, 16, true, false>) : BIOIK_NAMED_AS(PersistKernel, k_persist<1, 4, 1, false, 6, false, 16, true, false>);
#endif
}

} // namespace bioik
