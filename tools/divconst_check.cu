// Exhaustive check (all 2^32 fp32 bit patterns; NaN and +-inf inputs are routed to the division by the guard) that  q = a*r; q' = fma(fma(-d, q, a), r, q)  with r = RN(1/d) equals the
// correctly rounded a / d for the constant divisors the exact kernels use.  nvcc -arch=sm_90a -O3 tools/divconst_check.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__global__ void k(float d, float r, unsigned long long* bad, uint32_t* first, float lo) {
  const uint64_t n = 1ull << 32;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const float a = __uint_as_float((uint32_t)i);
    const float ref = __fdiv_rn(a, d);
    const float q = __fmul_rn(a, r);
    float fast = __fmaf_rn(__fmaf_rn(-d, q, a), r, q);
    if (!(fabsf(a) >= lo) || isinf(a)) fast = ref;                      // guard: tiny / non-finite inputs take the division
    if (__float_as_uint(fast) != __float_as_uint(ref) && !(isnan(fast) && isnan(ref))) {
      if (atomicAdd(bad, 1ull) == 0) *first = (uint32_t)i;
    }
  }
}
int main() {
  unsigned long long* bad; uint32_t* first;
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaMalloc(&bad, 8); cudaMalloc(&first, 4);
  const float ds[] = {9.f, 25.f, 49.f, 81.f, 255.f, 0.45f, 1.05f};
  for (float lo : {0.0f, 1e-30f}) for (float d : ds) {
    cudaMemset(bad, 0, 8); cudaMemset(first, 0, 4);
    k<<<sms * 16, 256>>>(d, 1.0f / d, bad, first, lo);
    unsigned long long hb; uint32_t hf;
    cudaMemcpy(&hb, bad, 8, cudaMemcpyDeviceToHost); cudaMemcpy(&hf, first, 4, cudaMemcpyDeviceToHost);
    printf("{\"divisor\": %g, \"guard_below\": %g, \"mismatches\": %llu, \"first_bits\": \"0x%08x\"}\n", d, lo, hb, hf);
  }
  return 0;
}
