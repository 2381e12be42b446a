// Microbenchmark: issue rate of the integer ops the POA DP inner loop could be built from (sm_90a).
// Prints warp-instructions per clock per SM for each op at 4, 8, 16 warps per SM.
#include <cstdio>
#include <cuda_runtime.h>

template <int OP>
__device__ __forceinline__ unsigned op(unsigned a, unsigned b, unsigned c) {
    if (OP == 0) return __viaddmax_s16x2(a, b, c);
    if (OP == 1) return (unsigned)__viaddmax_s32((int)a, (int)b, (int)c);
    if (OP == 2) return __vmaxs2(a, c) + b;            // VIMNMX.S16x2? + IADD
    if (OP == 3) return (a + b) ^ c;                  // IADD3 + LOP3
    if (OP == 4) return __byte_perm(a, b, c);         // PRMT
    if (OP == 5) return (unsigned)max((int)a + (int)b, (int)c);  // compiler's choice
    if (OP == 6) return __vimax3_s16x2(a, b, c);          // VIMNMX.S16x2
    if (OP == 7) return __vadd2(a, b);                // packed add
    if (OP == 8) return __viaddmax_s16x2_relu(a, b, c);
    return a;
}

template <int OP>
__global__ void k(unsigned* out, int iters, unsigned seed) {
    unsigned x[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = seed + threadIdx.x * 17 + i;
    unsigned b = seed | 1, c = seed * 3;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) x[i] = op<OP>(x[i], b, c + i);
    }
    unsigned s = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) s ^= x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int OP>
void run(const char* name, int instr_per_op) {
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    const int sms = prop.multiProcessorCount;   // one block per SM
    unsigned* out;
    cudaMalloc(&out, sms * 1024 * 4);
    int clk_khz;
    cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
    for (int warps = 4; warps <= 32; warps *= 2) {
        int iters = 20000;
        k<OP><<<sms, warps * 32>>>(out, 100, 1);
        cudaDeviceSynchronize();
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        cudaEventRecord(e0);
        k<OP><<<sms, warps * 32>>>(out, iters, 1);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        double ops = (double)warps * iters * 8;  // warp-level ops per SM
        double clocks = ms * 1e-3 * clk_khz * 1e3;
        printf("%-34s warps/SM=%2d  %.3f ops/clk/SM  (%.2f clk per warp-op per SMSP; nominal clock %d MHz; ~%d SASS/op)\n",
               name, warps, ops / clocks, 4.0 * clocks / ops, clk_khz / 1000, instr_per_op);
    }
    cudaFree(out);
}

int main() {
    run<0>("__viaddmax_s16x2 (VIADDMNMX.S16x2)", 1);
    run<1>("__viaddmax_s32   (VIADDMNMX)", 1);
    run<6>("__vimax3_s16x2   (VIMNMX3.S16x2)", 1);
    run<7>("__vadd2", 1);
    run<2>("__vmaxs2 + add", 2);
    run<3>("IADD3 + LOP3", 2);
    run<4>("__byte_perm      (PRMT)", 1);
    run<5>("max(a+b,c) int32", 1);
    run<8>("__viaddmax_s16x2_relu", 1);
    return 0;
}
