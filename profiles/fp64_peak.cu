// fp64_peak.cu — measures the FP64 pipe peak of the GPU this runs on (the roofline denominator of bench.py).
//
// Independent DFMA chains on every SM: each thread carries ILP register accumulators through a long unrolled loop
// of fused multiply-adds, blocks fill all SMs at several occupancies, CUDA events time the launch on its stream
// after a warm-up.  Reported per variant: TFLOP/s (FMA = 2 flop), the SM clock derived from clock64() against
// globaltimer inside the same launch, and DFMA warp-instructions per cycle per SM sub-partition (0.5 = one
// instruction every two cycles = a 16-lane FP64 unit per sub-partition).  The same for a pure DADD stream and a
// DFMA/DADD/DMUL/DSETP mix in the proportions of the generation kernel.
//
// Build + run (done by __graft_entry__.build() / profiles/measure_fp64_peak.sh on the GPU box):
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o profiles/_bin/fp64_peak profiles/fp64_peak.cu
//   profiles/_bin/fp64_peak > profiles/fp64_peak.json
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x)                                                                                       \
    do                                                                                              \
    {                                                                                               \
        cudaError_t e_ = (x);                                                                       \
        if(e_ != cudaSuccess)                                                                       \
        {                                                                                           \
            fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_));                                \
            return 2;                                                                               \
        }                                                                                           \
    } while(0)

__device__ __forceinline__ unsigned long long gtimer()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// MODE 0: DFMA only; 1: DADD only; 2: generation-kernel mix per 13 instructions: 5 DFMA, 4 DADD, 2 DMUL, 2 DSETP(+select);
// MODE 3 / 4: one DFMA + one / two independent 32-bit integer multiply-adds per step (does an FP64 instruction leave its second
// issue cycle to another pipe, or does it hold the dispatch port for both cycles?)
template <int ILP, int MODE> __global__ void __launch_bounds__(256) k_chains(double* out, int iters, double a, double b, unsigned long long* clk)
{
    double acc[ILP];
    unsigned iacc[ILP], jacc[ILP];
#pragma unroll
    for(int k = 0; k < ILP; k++) iacc[k] = threadIdx.x + k, jacc[k] = threadIdx.x * 3 + k;
    const unsigned im = (unsigned)iters | 1u, ia = (unsigned)(a * 1e6) | 1u;
#pragma unroll
    for(int k = 0; k < ILP; k++) acc[k] = (double)(threadIdx.x + k) * 1e-3;
    const long long c0 = clock64();
    const unsigned long long t0 = gtimer();
    for(int it = 0; it < iters; it++)
    {
#pragma unroll
        for(int u = 0; u < 8; u++)
        {
#pragma unroll
            for(int k = 0; k < ILP; k++)
            {
                if(MODE == 0)
                    acc[k] = __fma_rn(acc[k], a, b);
                else if(MODE == 1)
                    acc[k] = __dadd_rn(acc[k], b);
                else if(MODE == 3 || MODE == 4)
                {
                    acc[k] = __fma_rn(acc[k], a, b);
                    iacc[k] = iacc[k] * im + ia; // IMAD: integer pipe, independent of the FP64 chain
                    if(MODE == 4) jacc[k] = jacc[k] * ia + im;
                }
                else
                {
                    // 13 FP64-pipe instructions
                    double x = acc[k];
                    x = __fma_rn(x, a, b);
                    x = __fma_rn(x, a, b);
                    x = __fma_rn(x, a, b);
                    x = __fma_rn(x, a, b);
                    x = __fma_rn(x, a, b);
                    x = __dadd_rn(x, b);
                    x = __dadd_rn(x, a);
                    x = __dadd_rn(x, b);
                    x = __dadd_rn(x, a);
                    x = __dmul_rn(x, a);
                    x = __dmul_rn(x, a);
                    if(x < a) x = a;
                    if(x > 1e300) x = b;
                    acc[k] = x;
                }
            }
        }
    }
    const long long c1 = clock64();
    const unsigned long long t1 = gtimer();
    double s = 0;
#pragma unroll
    for(int k = 0; k < ILP; k++) s += acc[k] + (double)(iacc[k] ^ jacc[k]);
    out[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = s;
    if(threadIdx.x == 0)
    {
        clk[2 * blockIdx.x] = (unsigned long long)(c1 - c0);
        clk[2 * blockIdx.x + 1] = t1 - t0;
    }
}

struct Result
{
    const char* name;
    int ilp, blocks_per_sm, threads;
    double ms, tflops, inst_per_cycle_smsp, sm_mhz;
};

template <int ILP, int MODE> int run(const char* name, int sms, int blocks_per_sm, int iters, cudaStream_t st, double* d_out, unsigned long long* d_clk, std::vector<Result>& res)
{
    const int threads = 256, blocks = sms * blocks_per_sm;
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    for(int w = 0; w < 3; w++) k_chains<ILP, MODE><<<blocks, threads, 0, st>>>(d_out, iters, 0.9999999, 1e-9, d_clk);
    CK(cudaStreamSynchronize(st));
    const int reps = 5;
    float best = 1e30f;
    for(int r = 0; r < reps; r++)
    {
        CK(cudaEventRecord(e0, st));
        k_chains<ILP, MODE><<<blocks, threads, 0, st>>>(d_out, iters, 0.9999999, 1e-9, d_clk);
        CK(cudaEventRecord(e1, st));
        CK(cudaEventSynchronize(e1));
        float ms;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        if(ms < best) best = ms;
    }
    CK(cudaGetLastError());
    std::vector<unsigned long long> clk(2 * blocks);
    CK(cudaMemcpy(clk.data(), d_clk, clk.size() * 8, cudaMemcpyDeviceToHost));
    double cyc = 0, ns = 0;
    for(int b = 0; b < blocks; b++) cyc += (double)clk[2 * b], ns += (double)clk[2 * b + 1];
    const double sm_mhz = cyc / ns * 1e3;
    const double per_thread_inst = (double)iters * 8 * ILP * (MODE == 2 ? 13 : 1); // FP64 instructions (MODE 3 / 4: the DFMAs; the integer ops ride along)
    const double flop_per_inst = (MODE == 0 || MODE >= 3) ? 2.0 : (MODE == 1 ? 1.0 : (5 * 2 + 4 + 2 + 0) / 13.0);
    const double total_inst_thread = per_thread_inst * blocks * threads;
    const double tflops = total_inst_thread * flop_per_inst / (best * 1e-3) / 1e12;
    const double warp_inst = total_inst_thread / 32.0;
    const double cycles = best * 1e-3 * sm_mhz * 1e6;
    const double ipc = warp_inst / (cycles * sms * 4.0);
    res.push_back(Result{name, ILP, blocks_per_sm, threads, best, tflops, ipc, sm_mhz});
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return 0;
}

int main(int argc, char** argv)
{
    int dev = argc > 1 ? atoi(argv[1]) : 0;
    CK(cudaSetDevice(dev));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, dev));
    const int sms = prop.multiProcessorCount;
    cudaStream_t st;
    CK(cudaStreamCreate(&st));
    double* d_out;
    unsigned long long* d_clk;
    CK(cudaMalloc(&d_out, (size_t)sms * 8 * 256 * 8));
    CK(cudaMalloc(&d_clk, (size_t)sms * 8 * 2 * 8));
    std::vector<Result> res;
    const int iters = 4096;
    int rc = 0;
    rc |= run<8, 0>("dfma", sms, 2, iters, st, d_out, d_clk, res);
    rc |= run<8, 0>("dfma", sms, 4, iters, st, d_out, d_clk, res);
    rc |= run<16, 0>("dfma", sms, 2, iters, st, d_out, d_clk, res);
    rc |= run<16, 0>("dfma", sms, 4, iters, st, d_out, d_clk, res);
    rc |= run<8, 0>("dfma", sms, 8, iters, st, d_out, d_clk, res);
    rc |= run<8, 1>("dadd", sms, 4, iters, st, d_out, d_clk, res);
    rc |= run<4, 2>("mix_5fma_4add_2mul_2setp", sms, 4, iters / 4, st, d_out, d_clk, res);
    rc |= run<8, 3>("dfma_plus_1_imad", sms, 4, iters, st, d_out, d_clk, res);
    rc |= run<8, 4>("dfma_plus_2_imad", sms, 4, iters, st, d_out, d_clk, res);
    if(rc) return rc;
    double peak = 0, peak_mhz = 0, peak_ipc = 0;
    for(auto& r : res)
        if(r.name[1] == 'f' && r.name[4] == 0 && r.tflops > peak) peak = r.tflops, peak_mhz = r.sm_mhz, peak_ipc = r.inst_per_cycle_smsp;
    printf("{\"device\": \"%s\", \"sm_count\": %d, \"fp64_tflops\": %.4f, \"sm_mhz_during_peak\": %.1f, \"dfma_warp_inst_per_cycle_per_smsp\": %.4f,\n", prop.name, sms, peak, peak_mhz, peak_ipc);
    printf(" \"nominal_tflops_at_that_clock\": %.4f, \"method\": \"independent DFMA chains, CUDA events on the launch stream, best of 5 after 3 warm-ups; clock = clock64/globaltimer inside the launch\",\n",
           sms * 64.0 * 2.0 * peak_mhz * 1e6 / 1e12);
    printf(" \"variants\": [\n");
    for(size_t i = 0; i < res.size(); i++)
    {
        const Result& r = res[i];
        printf("  {\"stream\": \"%s\", \"ilp\": %d, \"blocks_per_sm\": %d, \"threads\": %d, \"ms\": %.4f, \"tflops\": %.4f, \"warp_inst_per_cycle_per_smsp\": %.4f, \"sm_mhz\": %.1f}%s\n", r.name, r.ilp, r.blocks_per_sm,
               r.threads, r.ms, r.tflops, r.inst_per_cycle_smsp, r.sm_mhz, i + 1 < res.size() ? "," : "");
    }
    printf(" ]}\n");
    return 0;
}
