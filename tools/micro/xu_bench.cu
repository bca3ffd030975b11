// Per-SM throughput of the instructions the attention softmax leans on: MUFU.EX2, F2FP (fp32x2 → bf16x2 pack), FFMA.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/micro/xu_bench tools/micro/xu_bench.cu
#include <cstdio>
#include <cuda_runtime.h>

template <int OP>
__global__ void k(float* out, int iters, float seed) {
  float a[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = seed + i * 0.01f + threadIdx.x * 1e-6f;
  unsigned acc = 0;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (OP == 0) {
        asm volatile("ex2.approx.ftz.f32 %0, %0;" : "+f"(a[i]));
      } else if (OP == 1) {
        unsigned r;
        asm volatile("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(a[i]), "f"(a[(i + 1) & 7]));
        acc ^= r;
      } else if (OP == 2) {
        asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(a[i]) : "f"(1.0001f), "f"(0.5f));
      } else if (OP == 3) {  // exp2 + pack, as in the softmax inner loop
        asm volatile("ex2.approx.ftz.f32 %0, %0;" : "+f"(a[i]));
        if (i & 1) {
          unsigned r;
          asm volatile("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(a[i]), "f"(a[i - 1]));
          acc ^= r;
        }
      } else if (OP == 4) {  // Cody-Waite style exp2 on the FMA pipe: floor + degree-3 polynomial + exponent insert
        float x = a[i];
        float fl = floorf(x);
        float f = x - fl;
        float p = fmaf(fmaf(fmaf(0.0555041f, f, 0.2402265f), f, 0.6931472f), f, 1.0f);
        int e = (int)fl;
        a[i] = __int_as_float(__float_as_int(p) + (e << 23)) * 1e-3f;
      } else if (OP == 5) {  // same, but rounding with the 1.5·2^23 magic constant: FADD/FFMA/SHL/IADD only (no XU-pipe conversion)
        float x = a[i];
        float t = x + 12582912.f;
        float fl = t - 12582912.f;
        float f = x - fl;  // [-0.5, 0.5]
        float p = fmaf(fmaf(fmaf(fmaf(0.0096181f, f, 0.0555041f), f, 0.2402265f), f, 0.6931472f), f, 1.0f);
        a[i] = __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23)) * 1e-3f;
      }
    }
  }
  float s = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += a[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s + (float)acc;
}

template <int OP>
void run(const char* name, int ops_per_iter) {
  int dev = 0, sms = 0, khz = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, dev);
  const int threads = 512, blocks = sms * 4, iters = 20000;
  float* out;
  cudaMalloc(&out, sizeof(float) * threads * blocks);
  k<OP><<<blocks, threads>>>(out, 100, 0.1f);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventRecord(e0);
  k<OP><<<blocks, threads>>>(out, iters, 0.1f);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  const double total = (double)blocks * threads * iters * ops_per_iter;
  const double per_s = total / (ms * 1e-3);
  // report per SM per clock at the MAX clock (the real clock under this load is lower, so this is a slight underestimate)
  printf("{\"op\": \"%s\", \"ms\": %.3f, \"Gops_per_s\": %.1f, \"ops_per_clk_per_sm_at_%dMHz\": %.2f}\n", name, ms, per_s / 1e9, khz / 1000,
         per_s / sms / (khz * 1e3));
  cudaFree(out);
}

int main() {
  run<0>("MUFU.EX2", 8);
  run<1>("F2FP.BF16 pack (cvt.rn.bf16x2.f32)", 8);
  run<2>("FFMA", 8);
  run<3>("EX2 x8 + F2FP x4 (softmax mix, counted as 8)", 8);
  run<4>("polynomial exp2 with FRND/F2I (counted as 8 exp2)", 8);
  run<5>("polynomial exp2, magic-constant rounding, FMA/ALU pipes only (counted as 8 exp2)", 8);
  return 0;
}
