// intra_plan_emul.cu — TEST INFRASTRUCTURE: exports the host function that builds k_intra's small-TU prediction plans
// (intra_plan_words in libde265_b200/csrc/kernels_recon.cuh, the very code engine.cu's init_tables runs to fill g_intra_plan)
// and the constants a plan word is read with.  tests/test_cpu_intra_plans.py executes the words with a restatement of
// tu_intra_fast's consumer and compares the result with the oracle's intra prediction, class by class, without a GPU.
// Built by tests/test_cpu_intra_plans.py with nvcc as a host-only shared library (tests/libintra_plan_emul.so); not part of
// the product.
#include <cstdint>

#include "kernels_recon.cuh"

#define EXPORT extern "C" __attribute__((visibility("default")))

EXPORT int intra_plan_classes() { return INTRA_PLAN_CLASSES; }
EXPORT int intra_plan_tile_stride() { return RC_TILE_STRIDE; }

// out[2]: the words of pixel slots 0 and 1 (pixels lane and lane + 32) of class cls.  Returns -1 for arguments out of range.
EXPORT int intra_plan_words(int cls, int lane, uint32_t* out)
{
  if (cls < 0 || cls >= INTRA_PLAN_CLASSES || lane < 0 || lane >= 32) return -1;
  void (*build)(int, int, uint32_t(&)[2]) = intra_plan_words;  // the header's function, not this wrapper
  uint32_t w[2];
  build(cls, lane, w);
  out[0] = w[0];
  out[1] = w[1];
  return 0;
}
