/* Plain-C consumer of the ControlNet entry points of include/sdxl_b200.h: they link against libsdxl_b200.so with the
 * prototypes of the header, and NULL objects are refused without touching a GPU. Built and run by tests/test_controlnet_cpu.py. */
#include <stddef.h>
#include <stdio.h>

#include "sdxl_b200.h"

int main(void) {
  int (*load)(sdxl_ctx*, const sdxl_controlnet_cfg*, const void*, size_t, int, sdxl_controlnet**) = sdxl_controlnet_load;
  void (*destroy)(sdxl_controlnet*) = sdxl_controlnet_destroy;
  int (*set)(sdxl_unet*, int, const sdxl_control*) = sdxl_unet_set_controls;
  int (*embed)(sdxl_controlnet*, int, int, int, const float*, int, float*) = sdxl_controlnet_embed_hint;
  sdxl_control c[SDXL_MAX_CONTROLS];
  sdxl_controlnet* net = NULL;
  c[0].net = NULL; c[0].hint = NULL; c[0].hint_on_host = 1; c[0].n_hint = 1; c[0].height = 8; c[0].width = 8; c[0].scale = 1.0f;
  if (load(NULL, NULL, NULL, 0, 0, &net) == 0 || set(NULL, 1, c) == 0 || embed(NULL, 1, 8, 8, NULL, 1, NULL) == 0) return 3;
  destroy(NULL);
  if (offsetof(sdxl_control, hint) != sizeof(void*) || offsetof(sdxl_control, scale) != offsetof(sdxl_control, width) + 4) return 4;
  if (offsetof(sdxl_controlnet_cfg, hint_in_channels) != sizeof(sdxl_unet_cfg)) return 5;
  printf("controlnet_abi_check ok %d %zu %zu\n", SDXL_MAX_CONTROLS, sizeof(sdxl_control), sizeof(sdxl_controlnet_cfg));
  return 0;
}
