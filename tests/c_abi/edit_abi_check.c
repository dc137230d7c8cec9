/* Plain-C consumer of the instruction-editing entry point of include/sdxl_b200.h: it links against libsdxl_b200.so with the prototype of
 * the header, and a NULL UNet is refused without touching a GPU. Prints sizeof(sdxl_edit_image), offsetof(sdxl_unet_cfg, edit_layout)
 * and sizeof(sdxl_unet_cfg) for tests/test_edit_cpu.py to compare with the ctypes mirror. */
#include <stddef.h>
#include <stdio.h>

#include "sdxl_b200.h"

int main(void) {
  int (*set)(sdxl_unet*, const sdxl_edit_image*) = sdxl_unet_set_edit_image;
  sdxl_edit_image e;
  e.latent = NULL; e.on_host = 1; e.n = 1; e.height = 64; e.width = 64; e.image_guidance = 1.5f;
  if (set(NULL, &e) == 0 || set(NULL, NULL) == 0) return 3;
  if (offsetof(sdxl_edit_image, on_host) != sizeof(void*) || offsetof(sdxl_edit_image, image_guidance) != offsetof(sdxl_edit_image, width) + 4)
    return 4;
  if (offsetof(sdxl_unet_cfg, edit_layout) != offsetof(sdxl_unet_cfg, n_steps) + 4) return 5;
  printf("edit_abi_check ok %zu %zu %zu\n", sizeof(sdxl_edit_image), offsetof(sdxl_unet_cfg, edit_layout), sizeof(sdxl_unet_cfg));
  return 0;
}
