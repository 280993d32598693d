// torch_stream.cpp — TEST INFRASTRUCTURE.  The torch-stream index mapping and counter / key layout of
// comfyui-vrgamedevgirl_b200/csrc/vrgdg_math.cuh compiled for the host with g++ (tests/test_torch_stream_cpu.py compares them
// with a restatement of ATen's launch policy and grid-stride loop).  Never loaded by the product.
#include "../../comfyui-vrgamedevgirl_b200/csrc/vrgdg_math.cuh"
#include <stdint.h>

using namespace vrgdg;

extern "C" {

uint32_t ts_threads(uint64_t numel, int sms, int max_threads_per_sm) { return torch_randn_threads(numel, sms, max_threads_per_sm); }

// elements li0 .. li0+n-1 of a draw of T threads -> (k, ii, idx) each
void ts_sites(uint32_t li0, uint32_t n, uint32_t T, uint32_t* k, uint32_t* ii, uint32_t* idx) {
  for (uint32_t i = 0; i < n; ++i) {
    const TorchSite s = torch_randn_site(li0 + i, T);
    k[i] = s.k; ii[i] = s.ii; idx[i] = s.idx;
  }
}

// the 128 bits behind element li of a draw seeded `seed`
void ts_bits(uint64_t seed, uint32_t li, uint32_t T, uint32_t* out) {
  const U4 r = torch_randn_bits(seed, torch_randn_site(li, T));
  out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
}

void ts_philox(const uint32_t* ctr, const uint32_t* key, uint32_t* out) {
  const U4 r = philox4x32_10(U4{ctr[0], ctr[1], ctr[2], ctr[3]}, key[0], key[1]);
  out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
}

uint64_t ts_draw_seed(uint64_t seed, int64_t frame0, int64_t i, int mode) { return torch_draw_seed(seed, frame0, i, mode); }
uint32_t ts_draw_base(int64_t i, int64_t hw, int mode) { return torch_draw_base(i, hw, mode); }

}  // extern "C"
