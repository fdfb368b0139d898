// The NTT pass planner (ntt_make_plan, ntt.cuh) compiled for the host (TEST ONLY), so that the planner's restatement
// in tests/ntt_cases.py can be pinned to it.  Used by tests/test_ntt_plans_emulation.py; NOT loaded by the product.
#include "ntt.cuh"

using namespace gb200;

extern "C" {

// ntt_make_plan(logn, tile_log) as out = {npasses, lo_bit, S, cb of pass 0, of pass 1, ...} (1 + 3 * NTT_MAX_PASSES ints)
int emu_ntt_plan(int logn, int tile_log, int* out) {
  const NttPlan pl = ntt_make_plan(logn, tile_log);
  out[0] = pl.npasses;
  for (int p = 0; p < pl.npasses; p++) {
    out[1 + 3 * p] = pl.pass[p].lo_bit;
    out[2 + 3 * p] = pl.pass[p].S;
    out[3 + 3 * p] = pl.pass[p].cb;
  }
  return 0;
}

}  // extern "C"
