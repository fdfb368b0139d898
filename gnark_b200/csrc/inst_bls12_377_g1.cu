// bls12_377: G1 MSM and group-NTT kernels (see inst.cuh)
#include "inst.cuh"
namespace gb200 {
GB200_REGISTER_MSM_G1(bls12_377_g1, 2, bls12_377_fr, bls12_377_fp)
}  // namespace gb200
