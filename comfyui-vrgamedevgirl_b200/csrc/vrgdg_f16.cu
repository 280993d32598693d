// kernels and launchers for __half frames
#include "vrgdg_inst.cuh"
namespace vrgdg {
VRGDG_INSTANTIATE(__half)
VRGDG_INSTANTIATE_CODECS(__half)
VRGDG_INSTANTIATE_FLOAT(__half)
}
