// microbench.cu -- pipe-throughput probes for H100 (sm_90a): lane-ops per clock per SM for the arithmetic the kernels
// lean on.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/microbench tools/microbench.cu
#include <cstdio>
#include <cuda_runtime.h>

template <int OP>
__global__ void probe(double *out, int iters, double seed) {
    double a0 = seed + threadIdx.x, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
    float f0 = (float)a0, f1 = f0 + 1, f2 = f0 + 2, f3 = f0 + 3, f4 = f0 + 4, f5 = f0 + 5, f6 = f0 + 6, f7 = f0 + 7;
    const double c = seed * 1e-9 + 1.0;
    const float cf = (float)c;
    unsigned long long p0, p1, p2, p3, p4, p5, p6, p7, pc;
    asm("mov.b64 %0, {%1, %2};" : "=l"(p0) : "f"(f0), "f"(f1)); asm("mov.b64 %0, {%1, %2};" : "=l"(p1) : "f"(f2), "f"(f3));
    asm("mov.b64 %0, {%1, %2};" : "=l"(p2) : "f"(f4), "f"(f5)); asm("mov.b64 %0, {%1, %2};" : "=l"(p3) : "f"(f6), "f"(f7));
    asm("mov.b64 %0, {%1, %2};" : "=l"(p4) : "f"(f1), "f"(f2)); asm("mov.b64 %0, {%1, %2};" : "=l"(p5) : "f"(f3), "f"(f4));
    asm("mov.b64 %0, {%1, %2};" : "=l"(p6) : "f"(f5), "f"(f6)); asm("mov.b64 %0, {%1, %2};" : "=l"(p7) : "f"(f7), "f"(f0));
    asm("mov.b64 %0, {%1, %2};" : "=l"(pc) : "f"(cf), "f"(cf));
    for (int i = 0; i < iters; i++) {
        if (OP == 0) { a0 = __dadd_rn(a0, c); a1 = __dadd_rn(a1, c); a2 = __dadd_rn(a2, c); a3 = __dadd_rn(a3, c); a4 = __dadd_rn(a4, c); a5 = __dadd_rn(a5, c); a6 = __dadd_rn(a6, c); a7 = __dadd_rn(a7, c); }
        if (OP == 1) { a0 = __dmul_rn(a0, c); a1 = __dmul_rn(a1, c); a2 = __dmul_rn(a2, c); a3 = __dmul_rn(a3, c); a4 = __dmul_rn(a4, c); a5 = __dmul_rn(a5, c); a6 = __dmul_rn(a6, c); a7 = __dmul_rn(a7, c); }
        if (OP == 2) { a0 = __fma_rn(a0, c, c); a1 = __fma_rn(a1, c, c); a2 = __fma_rn(a2, c, c); a3 = __fma_rn(a3, c, c); a4 = __fma_rn(a4, c, c); a5 = __fma_rn(a5, c, c); a6 = __fma_rn(a6, c, c); a7 = __fma_rn(a7, c, c); }
        if (OP == 3) { f0 = __fadd_rn(f0, cf); f1 = __fadd_rn(f1, cf); f2 = __fadd_rn(f2, cf); f3 = __fadd_rn(f3, cf); f4 = __fadd_rn(f4, cf); f5 = __fadd_rn(f5, cf); f6 = __fadd_rn(f6, cf); f7 = __fadd_rn(f7, cf); }
        if (OP == 4) { f0 = __fmul_rn(f0, cf); f1 = __fmul_rn(f1, cf); f2 = __fmul_rn(f2, cf); f3 = __fmul_rn(f3, cf); f4 = __fmul_rn(f4, cf); f5 = __fmul_rn(f5, cf); f6 = __fmul_rn(f6, cf); f7 = __fmul_rn(f7, cf); }
        if (OP == 5) { f0 = __fmaf_rn(f0, cf, cf); f1 = __fmaf_rn(f1, cf, cf); f2 = __fmaf_rn(f2, cf, cf); f3 = __fmaf_rn(f3, cf, cf); f4 = __fmaf_rn(f4, cf, cf); f5 = __fmaf_rn(f5, cf, cf); f6 = __fmaf_rn(f6, cf, cf); f7 = __fmaf_rn(f7, cf, cf); }
#define P2(op, r) asm volatile(op " %0, %0, %1;" : "+l"(r) : "l"(pc))
        if (OP == 6) { P2("add.rn.f32x2", p0); P2("add.rn.f32x2", p1); P2("add.rn.f32x2", p2); P2("add.rn.f32x2", p3); P2("add.rn.f32x2", p4); P2("add.rn.f32x2", p5); P2("add.rn.f32x2", p6); P2("add.rn.f32x2", p7); }
        if (OP == 7) { P2("mul.rn.f32x2", p0); P2("mul.rn.f32x2", p1); P2("mul.rn.f32x2", p2); P2("mul.rn.f32x2", p3); P2("mul.rn.f32x2", p4); P2("mul.rn.f32x2", p5); P2("mul.rn.f32x2", p6); P2("mul.rn.f32x2", p7); }
#define P3(r) asm volatile("fma.rn.f32x2 %0, %0, %1, %1;" : "+l"(r) : "l"(pc))
        if (OP == 8) { P3(p0); P3(p1); P3(p2); P3(p3); P3(p4); P3(p5); P3(p6); P3(p7); }
        if (OP == 9) { // DSETP + select chain
            a0 = a0 < c ? a1 : a0 + 1e-300; a2 = a2 < c ? a3 : a2; a4 = a4 < c ? a5 : a4; a6 = a6 < c ? a7 : a6;
            a1 = a1 < c ? a0 : a1; a3 = a3 < c ? a2 : a3; a5 = a5 < c ? a4 : a5; a7 = a7 < c ? a6 : a7;
        }
    }
    float q0, q1;
    asm("mov.b64 {%0, %1}, %2;" : "=f"(q0), "=f"(q1) : "l"(p0 ^ p1 ^ p2 ^ p3 ^ p4 ^ p5 ^ p6 ^ p7));
    out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7 + f0 + f1 + f2 + f3 + f4 + f5 + f6 + f7 + q0 + q1;
}

template <int OP>
void run(const char *name, int lanes_per_instr) {
    int dev; cudaGetDevice(&dev); cudaDeviceProp p; cudaGetDeviceProperties(&p, dev);
    const int blocks = p.multiProcessorCount * 4, threads = 256, iters = 20000;
    double *out; cudaMalloc(&out, sizeof(double) * blocks * threads);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    probe<OP><<<blocks, threads>>>(out, 1000, 1.0); cudaDeviceSynchronize();
    cudaEventRecord(e0); probe<OP><<<blocks, threads>>>(out, iters, 1.0); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    int clk; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, dev);
    const double ops = (double)blocks * threads * iters * 8.0 * lanes_per_instr;
    printf("%-22s %8.3f ms  %8.2f Gop/s  %7.2f lane-ops/clk/SM (at max clock %d MHz)\n", name, ms, ops / ms / 1e6,
           ops / (ms * 1e-3) / p.multiProcessorCount / (clk * 1e3), clk / 1000);
    cudaFree(out);
}

int main() {
    run<0>("DADD", 1); run<1>("DMUL", 1); run<2>("DFMA", 1); run<9>("DSETP+SEL (x1)", 1);
    run<3>("FADD", 1); run<4>("FMUL", 1); run<5>("FFMA", 1);
    run<6>("add.f32x2", 2); run<7>("mul.f32x2", 2); run<8>("fma.f32x2", 2);
    return 0;
}
