/* Plain-C consumer of the FreeU entry point of include/sdxl_b200.h: it links against libsdxl_b200.so with the prototype of the header,
 * and a NULL UNet is refused without touching a GPU. Built and run by tests/test_freeu_cpu.py. */
#include <stddef.h>
#include <stdio.h>

#include "sdxl_b200.h"

int main(void) {
  int (*set)(sdxl_unet*, const sdxl_freeu*) = sdxl_unet_set_freeu;
  sdxl_freeu f;
  f.s1 = 0.9f; f.s2 = 0.2f; f.b1 = 1.3f; f.b2 = 1.4f;
  if (set(NULL, &f) == 0 || set(NULL, NULL) == 0) return 3;
  if (offsetof(sdxl_freeu, s2) != 4 || offsetof(sdxl_freeu, b1) != 8 || offsetof(sdxl_freeu, b2) != 12) return 4;
  printf("freeu_abi_check ok %zu\n", sizeof(sdxl_freeu));
  return 0;
}
