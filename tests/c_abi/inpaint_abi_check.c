/* Plain-C consumer of the inpainting entry point of include/sdxl_b200.h: it links against libsdxl_b200.so with the prototype of the
 * header, and a NULL UNet is refused without touching a GPU. Built and run by tests/test_inpaint_cpu.py. */
#include <stddef.h>
#include <stdio.h>

#include "sdxl_b200.h"

int main(void) {
  int (*set)(sdxl_unet*, const sdxl_inpaint_condition*) = sdxl_unet_set_inpaint_condition;
  sdxl_inpaint_condition c;
  c.cond = NULL; c.on_host = 1; c.n = 1; c.height = 64; c.width = 64;
  if (set(NULL, &c) == 0 || set(NULL, NULL) == 0) return 3;
  if (offsetof(sdxl_inpaint_condition, on_host) != sizeof(void*) || offsetof(sdxl_inpaint_condition, width) != offsetof(sdxl_inpaint_condition, height) + 4)
    return 4;
  printf("inpaint_abi_check ok %zu\n", sizeof(sdxl_inpaint_condition));
  return 0;
}
