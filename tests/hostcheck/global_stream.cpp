// global_stream.cpp — TEST INFRASTRUCTURE.  The global-generator draw geometry, Philox offset and counter increment of
// comfyui-vrgamedevgirl_b200/csrc/vrgdg_math.cuh compiled for the host with g++ (tests/test_global_stream_cpu.py compares them with
// a restatement of the reference's mini-batch loop, ATen's launch policy and curand's skipahead).  Never loaded by the product.
#include "../../comfyui-vrgamedevgirl_b200/csrc/vrgdg_math.cuh"
#include <stdint.h>

using namespace vrgdg;

extern "C" {

uint32_t gs_threads(uint64_t numel, int sms, int max_threads_per_sm) { return torch_randn_threads(numel, sms, max_threads_per_sm); }

void gs_philox(const uint32_t* ctr, const uint32_t* key, uint32_t* out) {
  const U4 r = philox4x32_10(U4{ctr[0], ctr[1], ctr[2], ctr[3]}, key[0], key[1]);
  out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
}

// the 128 bits behind element li of a draw seeded `seed` at Philox offset `offset` (a multiple of 4); offset 0 = a fresh generator
void gs_bits_at(uint64_t seed, uint32_t li, uint32_t T, uint64_t offset, uint32_t* out) {
  const U4 r = torch_randn_bits(seed, torch_randn_site(li, T), offset / 4);
  out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
}

// the same bits through the fresh-generator call the per-frame / per-call modes make (no offset argument)
void gs_bits_fresh(uint64_t seed, uint32_t li, uint32_t T, uint32_t* out) {
  const U4 r = torch_randn_bits(seed, torch_randn_site(li, T));
  out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
}

uint64_t gs_increment(uint64_t numel, uint32_t T) { return torch_randn_increment<uint64_t>(numel, T); }

// the global generator's draw of absolute frame f: {draw j, element base, numel_j, T_j, offset o_j}
void gs_global_draw(uint32_t f, uint32_t step, uint32_t clip, uint32_t n, uint32_t T_full, uint32_t T_last, uint64_t o0, uint64_t* out) {
  const uint32_t j = torch_global_draw(f, step);
  out[0] = j;
  out[1] = torch_global_base(f, step, n);
  out[2] = torch_global_numel(j, step, clip, n);
  out[3] = torch_global_threads(j, step, clip, T_full, T_last);
  out[4] = torch_global_offset(o0, j, step, n, T_full);
}

}  // extern "C"
