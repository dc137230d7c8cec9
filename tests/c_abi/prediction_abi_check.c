/* Plain-C consumer of the prediction entry point of include/sdxl_b200.h: it links against libsdxl_b200.so with the prototype of the
 * header, and a NULL UNet is refused without touching a GPU. Built and run by tests/test_prediction_cpu.py. */
#include <stddef.h>
#include <stdio.h>

#include "sdxl_b200.h"

int main(void) {
  int (*set)(sdxl_unet*, const sdxl_prediction*) = sdxl_unet_set_prediction;
  static const double table[2] = {0.5, 0.25};
  sdxl_prediction p;
  p.type = SDXL_PREDICTION_V; p.guidance_rescale = 0.7f; p.n_alphas = 2; p.alphas_cumprod_host = table;
  if (set(NULL, &p) == 0 || set(NULL, NULL) == 0) return 3;
  if (SDXL_PREDICTION_EPSILON != 0 || SDXL_PREDICTION_V != 1) return 4;
  if (offsetof(sdxl_prediction, guidance_rescale) != 4 || offsetof(sdxl_prediction, n_alphas) != 8 ||
      offsetof(sdxl_prediction, alphas_cumprod_host) != 16)
    return 5;
  printf("prediction_abi_check ok %zu\n", sizeof(sdxl_prediction));
  return 0;
}
