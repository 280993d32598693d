// global_noise.cpp — TEST INFRASTRUCTURE.  The work-item -> element mapping of k_torch_global_noise (torch_global_window,
// torch_global_item, torch_global_li in comfyui-vrgamedevgirl_b200/csrc/vrgdg_math.cuh) compiled for the host with g++:
// tests/test_postchain_global_stream_cpu.py walks every work item of a window and checks what each one stores.  Never loaded by the
// product.
#include "../../comfyui-vrgamedevgirl_b200/csrc/vrgdg_math.cuh"
#include <stdint.h>

using namespace vrgdg;

extern "C" {

// Every store the kernel makes for frames [frame0, frame0 + frames) of a clip: visits[e] counts the stores to element e of the
// window's [frames, n] tensor, site[3 e .. 3 e + 2] = the (k, ii, idx) of the last one and draw[e] its draw.  The work items are
// those of the launch: rows r < w.rows, idx < T_full (idx >= T_j stores nothing).  Returns the number of rows, 0 when the window
// has more than `max_rows` of them.
uint32_t gn_walk(uint32_t frame0, uint32_t frames, uint32_t n, uint32_t step, uint32_t clip, uint32_t T_full, uint32_t T_last,
                 uint32_t max_rows, uint32_t* visits, uint32_t* site, uint32_t* draw) {
  const TorchGlobalWindow w = torch_global_window(frame0, frames, n, step, clip, T_full, T_last);
  if (w.rows > max_rows) return 0;
  for (uint32_t r = 0; r < w.rows; ++r) {
    for (uint32_t idx = 0; idx < T_full; ++idx) {
      TorchGlobalItem it;
      if (!torch_global_item(w, r, idx, it)) continue;
      for (uint32_t ii = 0; ii < 4; ++ii) {
        const uint32_t li = torch_global_li(it, idx, ii);
        if (li < it.lo || li >= it.hi) continue;
        const int64_t e = it.base + li;
        visits[e] += 1;
        site[3 * e] = it.k; site[3 * e + 1] = ii; site[3 * e + 2] = idx;
        draw[e] = it.j;
      }
    }
  }
  return w.rows;
}

// torch_randn_site of elements li[i] of draws of T[i] threads: out[3 i ..] = {k, ii, idx}
void gn_sites(const uint32_t* li, const uint32_t* T, uint64_t count, uint32_t* out) {
  for (uint64_t i = 0; i < count; ++i) {
    const TorchSite s = torch_randn_site(li[i], T[i]);
    out[3 * i] = s.k; out[3 * i + 1] = s.ii; out[3 * i + 2] = s.idx;
  }
}

uint32_t gn_threads(uint64_t numel, int sms, int max_threads_per_sm) { return torch_randn_threads(numel, sms, max_threads_per_sm); }

}  // extern "C"
