// kernels and launchers for __nv_bfloat16 frames
#include "vrgdg_inst.cuh"
namespace vrgdg {
VRGDG_INSTANTIATE(__nv_bfloat16)
VRGDG_INSTANTIATE_CODECS(__nv_bfloat16)
VRGDG_INSTANTIATE_FLOAT(__nv_bfloat16)
}
