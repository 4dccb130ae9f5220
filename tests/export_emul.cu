// export_emul.cu — TEST INFRASTRUCTURE: the RGB export's coefficient derivation and per-pixel function
// (libde265_b200/csrc/export.cuh, the same functions the GPU executes) built for the host.  Used by tests/test_cpu_export.py.
#include <cstdint>
#include "export.cuh"

// coefs[7] = {y, r_cr, g_cb, g_cr, b_cb, oy, oc}
extern "C" __attribute__((visibility("default"))) void export_emul_coefs(int matrix, int full_range, int bd_y, int bd_c, int* coefs)
{
  const ExportCoefs c = export_coefs(matrix, full_range != 0, bd_y, bd_c);
  const int v[7] = {c.y, c.r_cr, c.g_cb, c.g_cr, c.b_cb, c.oy, c.oc};
  for (int i = 0; i < 7; i++) coefs[i] = v[i];
}

// rgb[3 * i + o] for the samples (y[i], cb[i], cr[i])
extern "C" __attribute__((visibility("default"))) void export_emul_rgb(int matrix, int full_range, int bd_y, int bd_c, const int32_t* y,
                                                                       const int32_t* cb, const int32_t* cr, long n, uint8_t* rgb)
{
  const ExportCoefs c = export_coefs(matrix, full_range != 0, bd_y, bd_c);
  for (long i = 0; i < n; i++) export_rgb_pixel(c, y[i], cb[i], cr[i], rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]);
}
