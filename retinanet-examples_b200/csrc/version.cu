// version.cu -- library identification and the process-wide launch budget.
#include "common.cuh"
int g_odtk_sm_budget = 0;
extern "C" const char *odtk_b200_version(void) { return "odtk_b200 0.1 sm_90a"; }
// Persistent kernels launched after this call use at most `sms` CTAs (rounded down to an even number; 0 = all SMs of the
// device).  Host-side state read at launch time: a CUDA graph keeps the grid it was captured with.
extern "C" int odtk_set_sm_budget(int sms) {
  if (sms < 0) return ODTK_E_INVALID;
  g_odtk_sm_budget = sms & ~1;
  return ODTK_OK;
}
int g_odtk_tma_store = 1;
// fp16 NHWC convolution / bottleneck-tail outputs: TMA stores from shared memory (1) or direct stores (0); returns the
// previous setting.  Read at launch time, like the budget.
extern "C" int odtk_set_tma_store(int on) {
  const int prev = g_odtk_tma_store;
  g_odtk_tma_store = on != 0;
  return prev;
}
