// bls12_381: G1 MSM and group-NTT kernels (see inst.cuh)
#include "inst.cuh"
namespace gb200 {
GB200_REGISTER_MSM_G1(bls12_381_g1, 1, bls12_381_fr, bls12_381_fp)
}  // namespace gb200
