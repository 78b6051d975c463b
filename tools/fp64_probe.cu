// fp64 pipe probe (tool, not product): what does a DFMA/DMUL/DADD cost on sm_90 as a function of where its operands
// come from, and what is the dependent-issue latency?  The answers bound K1/K2 (DESIGN.md "what bounds K1").
//   pattern   SASS shape (checked with cuobjdump)              register-file reads per instruction
//   0 fma_ri  DFMA x, x, Ra.reuse, 0.5                         1 fresh pair
//   1 fma_rr  DFMA x, x, Ra.reuse, Rb.reuse                    1 fresh pair (two reuse-cache hits)
//   2 fma_2   DFMA x, x, y_k, 0.5          y_k distinct per k   2 fresh pairs
//   3 fma_3   DFMA x, x, y_k, z_k                               3 fresh pairs
//   4 mul_2   DMUL x, x, y_k                                    2 fresh pairs
//   5 add_2   DADD x, x, y_k                                    2 fresh pairs
//   6 fma_ur  DFMA x, x, UR, Rb.reuse  (kernel parameter)       1 fresh pair
//   7 mix     the K1 mix: per 8 instr 3 fma_3, 2 fma_2, 3 mul_2
//   8 fma+1i  one independent integer instruction (IMAD) per DFMA: does the integer op hide behind the DFMA's two
//   9 fma+2i  pipe cycles, or does every issued instruction cost an issue cycle of its own?
// `chains` independent accumulators per thread (ILP), `warps` per SM (TLP): chains=1 & 4 warps/SM exposes the latency.
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_probe tools/fp64_probe.cu
#include <cstdio>
#include <cuda_runtime.h>

static double *g_d, *g_in;
static int g_sms;

template <int kPat, int kChains>
__global__ void __launch_bounds__(256) probe(double *out, const double *in, int iters, double a) {
    double x[kChains], y[kChains], z[kChains];
#pragma unroll
    for (int k = 0; k < kChains; ++k) {
        x[k] = threadIdx.x * 1e-9 + k;
        y[k] = in[k] + threadIdx.x * 1e-13;   // thread-varying: must live in the register file, not in uniform registers
        z[k] = in[8 + k] - threadIdx.x * 1e-13;
    }
    double ra = in[16] + threadIdx.x * 1e-13, rb = in[17] - threadIdx.x * 1e-13;
#pragma unroll
    for (int k = 0; k < kChains; ++k) asm volatile("" : "+d"(y[k]), "+d"(z[k]));
    asm volatile("" : "+d"(ra), "+d"(rb));
#pragma unroll 1
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int r = 0; r < 64 / kChains; ++r) {
#pragma unroll
            for (int k = 0; k < kChains; ++k) {
                if (kPat == 0) x[k] = fma(x[k], ra, 0.5);
                if (kPat == 1) x[k] = fma(x[k], ra, rb);
                if (kPat == 2) x[k] = fma(x[k], y[k], 0.5);
                if (kPat == 3) x[k] = fma(x[k], y[k], z[k]);
                if (kPat == 4) x[k] = x[k] * y[k];
                if (kPat == 5) x[k] = x[k] + y[k];
                if (kPat == 6) x[k] = fma(x[k], a, rb);
                if (kPat == 7) {
                    const int q = (r * kChains + k) & 7;
                    if (q < 3) x[k] = fma(x[k], y[k], z[k]);
                    else if (q < 5) x[k] = fma(x[k], y[k], 0.5);
                    else x[k] = x[k] * y[k];
                }
            }
        }
    }
    double s = 0;
#pragma unroll
    for (int k = 0; k < kChains; ++k) s += x[k];
    if (s == 1234.5678) out[0] = s;
}

template <int kInts>
__global__ void __launch_bounds__(256) probe_int(double *out, const double *in, int iters, int m) {
    double x[8];
    int q[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        x[k] = threadIdx.x * 1e-9 + k;
        q[k] = threadIdx.x + k;
    }
    double ra = in[16] + threadIdx.x * 1e-13;
    asm volatile("" : "+d"(ra));
#pragma unroll 1
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int r = 0; r < 8; ++r) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                x[k] = fma(x[k], ra, 0.5);
                if (kInts >= 1) q[k] = q[k] * m + 12345;         // IMAD
                if (kInts >= 2) q[(k + 4) & 7] ^= (q[k] >> 3);    // SHF/LOP3
            }
        }
    }
    double s = 0;
    int t = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) { s += x[k]; t += q[k]; }
    if (s == 1234.5678 || t == 123456789) out[0] = s + t;
}

template <int kInts>
double run_int() {
    const int threads = 256, blocks = g_sms * 8, iters = 2048;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    float best = 1e30f;
    for (int rep = 0; rep < 6; ++rep) {
        cudaEventRecord(e0);
        probe_int<kInts><<<blocks, threads>>>(g_d, g_in, iters, 3);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        if (rep > 1 && ms < best) best = ms;
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return 64.0 * iters * (double)blocks * threads / (best * 1e-3);  // DFMAs per second
}

template <int kPat, int kChains>
double run(int warpsPerSm) {
    const int threads = warpsPerSm >= 8 ? 256 : warpsPerSm * 32;
    const int blocks = g_sms * (warpsPerSm >= 8 ? warpsPerSm / 8 : 1);
    const int iters = 2048;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    float best = 1e30f;
    for (int rep = 0; rep < 6; ++rep) {
        cudaEventRecord(e0);
        probe<kPat, kChains><<<blocks, threads>>>(g_d, g_in, iters, 0.999999);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        if (rep > 1 && ms < best) best = ms;
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    const double inst = 64.0 * iters * (double)blocks * threads;  // thread-level fp64 instructions
    return inst / (best * 1e-3);                                  // instructions per second
}

template <int kPat>
void row(const char *name, double clkHz) {
    // cycles per warp-instruction per SMSP = (SMSPs * clk) / (inst/s / 32)
    auto cyc = [&](double ips) { return g_sms * 4.0 * clkHz / (ips / 32.0); };
    const double full = run<kPat, 8>(64), c4w16 = run<kPat, 4>(16), c2w8 = run<kPat, 2>(8), lat = run<kPat, 1>(4);
    printf("{\"pattern\": \"%s\", \"Tinst_per_s_full\": %.3f, \"cycles_per_warp_instr_full\": %.3f, "
           "\"cycles_ilp4_4warps_per_smsp\": %.3f, \"cycles_ilp2_2warps_per_smsp\": %.3f, "
           "\"dependent_issue_latency_cycles\": %.2f}\n",
           name, full * 1e-12, cyc(full), cyc(c4w16), cyc(c2w8), cyc(lat));
}

int main() {
    cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0);
    int khz = 0;
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    const double clk = khz * 1e3;
    cudaMalloc(&g_d, 64);
    cudaMalloc(&g_in, 32 * 8);
    double h[32];
    for (int i = 0; i < 32; ++i) h[i] = 0.999999 + 1e-9 * i;
    cudaMemcpy(g_in, h, sizeof h, cudaMemcpyHostToDevice);
    for (int warm = 0; warm < 20; ++warm) run<0, 8>(64);
    printf("{\"sms\": %d, \"clock_mhz\": %.0f, \"pipe_peak_Tinst\": %.3f}\n", g_sms, clk * 1e-6, g_sms * 64.0 * clk * 1e-12);
    row<0>("fma x,Ra.reuse,imm (1 fresh pair)", clk);
    row<1>("fma x,Ra.reuse,Rb.reuse", clk);
    row<6>("fma x,UR,Rb.reuse", clk);
    row<2>("fma x,y_k,imm (2 fresh pairs)", clk);
    row<3>("fma x,y_k,z_k (3 fresh pairs)", clk);
    row<4>("mul x,y_k (2 fresh pairs)", clk);
    row<5>("add x,y_k (2 fresh pairs)", clk);
    row<7>("K1 mix 3:2:3 fma3:fma2:mul2", clk);
    {
        auto cyc = [&](double ips) { return g_sms * 4.0 * clk / (ips / 32.0); };
        printf("{\"pattern\": \"DFMA alone / +1 integer instr / +2-3 integer instrs, per DFMA\", \"cycles_per_dfma\": [%.3f, %.3f, %.3f]}\n",
               cyc(run_int<0>()), cyc(run_int<1>()), cyc(run_int<2>()));
    }
    return 0;
}
