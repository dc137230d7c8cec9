/* Plain-C consumer of the T2I-Adapter entry points of include/sdxl_b200.h: they link against libsdxl_b200.so with the prototypes
 * of the header, and NULL objects are refused without touching a GPU. Built and run by tests/test_t2i_adapter_cpu.py. */
#include <stddef.h>
#include <stdio.h>

#include "sdxl_b200.h"

int main(void) {
  int (*load)(sdxl_ctx*, const sdxl_t2i_adapter_cfg*, const void*, size_t, int, sdxl_t2i_adapter**) = sdxl_t2i_adapter_load;
  void (*destroy)(sdxl_t2i_adapter*) = sdxl_t2i_adapter_destroy;
  int (*set)(sdxl_unet*, int, const sdxl_t2i_control*, int32_t) = sdxl_unet_set_t2i_adapters;
  int (*features)(sdxl_t2i_adapter*, int, int, int, const float*, int, float*) = sdxl_t2i_adapter_features;
  sdxl_t2i_control c[SDXL_MAX_T2I_ADAPTERS];
  sdxl_t2i_adapter* a = NULL;
  c[0].adapter = NULL; c[0].hint = NULL; c[0].hint_on_host = 1; c[0].n_hint = 1; c[0].height = 32; c[0].width = 32; c[0].scale = 1.0f;
  if (load(NULL, NULL, NULL, 0, 0, &a) == 0 || set(NULL, 1, c, 0) == 0 || features(NULL, 1, 32, 32, NULL, 1, NULL) == 0) return 3;
  destroy(NULL);
  if (offsetof(sdxl_t2i_control, hint) != sizeof(void*) || offsetof(sdxl_t2i_control, scale) != offsetof(sdxl_t2i_control, width) + 4) return 4;
  if (offsetof(sdxl_t2i_adapter_cfg, in_channels) != sizeof(sdxl_unet_cfg)) return 5;
  printf("t2i_adapter_abi_check ok %d %zu %zu\n", SDXL_MAX_T2I_ADAPTERS, sizeof(sdxl_t2i_control), sizeof(sdxl_t2i_adapter_cfg));
  return 0;
}
