// bn254: G1 MSM and group-NTT kernels (see inst.cuh)
#include "inst.cuh"
namespace gb200 {
GB200_REGISTER_MSM_G1(bn254_g1, 0, bn254_fr, bn254_fp)
}  // namespace gb200
