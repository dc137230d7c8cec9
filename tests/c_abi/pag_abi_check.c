/* Plain-C consumer of the PAG entry points of include/sdxl_b200.h: it links against libsdxl_b200.so with the prototypes of the header,
 * and a NULL UNet is refused without touching a GPU. Built and run by tests/test_pag_cpu.py. */
#include <stddef.h>
#include <stdio.h>

#include "sdxl_b200.h"

int main(void) {
  int (*set)(sdxl_unet*, const sdxl_pag*) = sdxl_unet_set_pag;
  int (*count)(const sdxl_unet*) = sdxl_unet_num_self_attentions;
  const uint8_t layers[2] = {1, 0};
  sdxl_pag p;
  p.scale = 3.0f; p.adaptive_scale = 0.0f; p.n_layers = 2; p.layers_host = layers; p.forward_perturbed_rows = 0;
  if (set(NULL, &p) == 0 || set(NULL, NULL) == 0 || count(NULL) >= 0) return 3;
  if (offsetof(sdxl_pag, n_layers) != 8 || offsetof(sdxl_pag, layers_host) != 16 || offsetof(sdxl_pag, forward_perturbed_rows) != 24)
    return 4;
  printf("pag_abi_check ok %zu\n", sizeof(sdxl_pag));
  return 0;
}
