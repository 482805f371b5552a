// Host build of the tensor-core GEMM's work list (csrc/gemm_schedule.cuh) for tests/test_gemm_schedule_cpu.py.
// TEST INFRASTRUCTURE ONLY.
#include "../../auto_avsr_b200/csrc/gemm_schedule.cuh"

extern "C" int tc_emu_items(int tiles_m, int tiles_n, int splits, int cm, int cn) {
  return avsr::tc_cluster_items(tiles_m, tiles_n, splits, cm, cn);
}

// out = {tm, tn, split, valid}
extern "C" void tc_emu_work(int item, int crank, int tiles_m, int tiles_n, int cm, int cn, int* out) {
  const avsr::TcWork w = avsr::tc_work_item(item, crank, tiles_m, tiles_n, cm, cn);
  out[0] = w.tm; out[1] = w.tn; out[2] = w.split; out[3] = w.valid ? 1 : 0;
}
