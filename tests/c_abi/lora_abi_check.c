/* Plain-C consumer of the LoRA adapter entry points of include/sdxl_b200.h: they link against libsdxl_b200.so with the
 * prototypes of the header, and NULL models are refused without touching a GPU. Built and run by tests/test_lora_cpu.py. */
#include <stddef.h>
#include <stdio.h>

#include "sdxl_b200.h"

int main(void) {
  int (*set_unet)(sdxl_unet*, int, const sdxl_adapter*) = sdxl_unet_set_adapters;
  int (*set_clip)(sdxl_clip*, int, const sdxl_adapter*) = sdxl_clip_set_adapters;
  sdxl_adapter a[SDXL_MAX_ADAPTERS];
  a[0].pack = NULL; a[0].bytes = 0; a[0].pack_on_device = 0; a[0].scale = 1.0f;
  if (set_unet(NULL, 1, a) == 0 || set_clip(NULL, 0, a) == 0) return 3;
  if (offsetof(sdxl_adapter, bytes) != sizeof(void*) || offsetof(sdxl_adapter, scale) != offsetof(sdxl_adapter, pack_on_device) + 4) return 4;
  printf("lora_abi_check ok %d %zu\n", SDXL_MAX_ADAPTERS, sizeof(sdxl_adapter));
  return 0;
}
