// Issue rate of the integer instructions the extractor kernels are made of (IMAD, IDP, VABSDIFF4, IADD3, LOP3, PRMT, SHF, VIMNMX3, POPC) on sm_90a: 8 independent chains per thread, 1024 threads per CTA, one CTA per SM.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o idp_rate idp_rate.cu && ./idp_rate
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

template <int OP>
__global__ void k(uint32_t* out, uint32_t seed, int iters, long long* cycles) {
    uint32_t a[8], b = seed | 0x01020304u;
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = seed + threadIdx.x * 8 + i;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (OP == 0) a[i] = a[i] * b + 7u;                                   // IMAD
            else if (OP == 1) a[i] = __dp4a(a[i], b, a[i]);                      // IDP.4A.U8.U8
            else if (OP == 2) a[i] = __dp2a_lo(a[i], b, a[i]);                   // IDP.2A.LO.U16.U8
            else if (OP == 3) asm("vabsdiff4.u32.u32.u32.add %0, %1, %2, %0;" : "+r"(a[i]) : "r"(a[i] ^ 0x55u), "r"(b));   // VABSDIFF4 + accumulate
            else if (OP == 4) a[i] = a[i] + b + (uint32_t)it;                     // IADD3
            else if (OP == 5) a[i] = (a[i] & b) ^ (uint32_t)it;                   // LOP3
            else if (OP == 6) a[i] = __byte_perm(a[i], b, 0x5140u);               // PRMT
            else if (OP == 7) a[i] = __funnelshift_r(a[i], b, 8u);                // SHF
            else if (OP == 8) a[i] = __vimax3_u16x2(a[i], b, (uint32_t)it);       // VIMNMX3.U16x2 (DPX)
            else if (OP == 9) a[i] = __vminu2(a[i], b + (uint32_t)it);            // packed 16x2 min
            else if (OP == 10) a[i] = (uint32_t)__popc(a[i]) + b;                 // POPC (+ IADD)
            else a[i] = a[i] > b ? a[i] - b : a[i] + (uint32_t)it;                // ISETP + SEL / predicated adds
        }
    }
    const long long t1 = clock64();
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) s ^= a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int OP>
void run(const char* name, uint32_t* out, long long* cyc, int sms) {
    const int iters = 4096;
    k<OP><<<sms, 1024>>>(out, 3u, iters, cyc);
    k<OP><<<sms, 1024>>>(out, 3u, iters, cyc);
    cudaDeviceSynchronize();
    long long h[256];
    cudaMemcpy(h, cyc, sizeof(long long) * sms, cudaMemcpyDeviceToHost);
    double avg = 0;
    for (int i = 0; i < sms; ++i) avg += (double)h[i];
    avg /= sms;
    const double warp_instr = (double)iters * 8 * 32;   // per SM: 32 warps x 8 x iters
    printf("%-28s %.1f cycles per SM for %.0f warp instructions: %.2f warp instr / clk / SM\n", name, avg, warp_instr, warp_instr / avg);
}

int main() {
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    uint32_t* out; long long* cyc;
    cudaMalloc(&out, sizeof(uint32_t) * sms * 1024);
    cudaMalloc(&cyc, sizeof(long long) * 256);
    printf("SMs %d\n", sms);
    run<0>("IMAD", out, cyc, sms);
    run<1>("IDP.4A.U8.U8", out, cyc, sms);
    run<2>("IDP.2A.LO.U16.U8", out, cyc, sms);
    run<3>("VABSDIFF4.U8 + acc", out, cyc, sms);
    run<4>("IADD3", out, cyc, sms);
    run<5>("LOP3", out, cyc, sms);
    run<6>("PRMT", out, cyc, sms);
    run<7>("SHF (funnel shift)", out, cyc, sms);
    run<8>("VIMNMX3.U16x2 (max3)", out, cyc, sms);
    run<9>("__vminu2 (16x2 min)", out, cyc, sms);
    run<10>("POPC + IADD", out, cyc, sms);
    run<11>("compare + select", out, cyc, sms);
    return cudaGetLastError() != cudaSuccess;
}
