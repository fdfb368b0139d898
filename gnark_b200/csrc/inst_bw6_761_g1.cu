// bw6_761: G1 MSM and group-NTT kernels (see inst.cuh)
#include "inst.cuh"
namespace gb200 {
GB200_REGISTER_MSM_G1(bw6_761_g1, 3, bw6_761_fr, bw6_761_fp)
GB200_REGISTER_MSM(bw6_761_g2, 3, 2, bw6_761_fr, bw6_761_fp)  // BW6-761 G2 is over Fp too
}  // namespace gb200
