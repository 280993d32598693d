// kernels and launchers for float frames
#include "vrgdg_inst.cuh"
namespace vrgdg {
VRGDG_INSTANTIATE(float)
VRGDG_INSTANTIATE_CODECS(float)
VRGDG_INSTANTIATE_FLOAT(float)
}
