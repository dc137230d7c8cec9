/* Plain-C consumer of the image-prompt set entry point of include/sdxl_b200.h: it links against libsdxl_b200.so with the prototype
 * of the header, the limits are the documented ones, and a NULL UNet is refused without touching a GPU. Built and run by
 * tests/test_ip_multi_cpu.py. */
#include <stddef.h>
#include <stdio.h>
#include <string.h>

#include "sdxl_b200.h"

int main(void) {
  int (*set)(sdxl_unet*, int, const sdxl_image_prompt*, const sdxl_ip_mask*) = sdxl_unet_set_image_prompts;
  sdxl_image_prompt p[SDXL_MAX_IMAGE_PROMPTS];
  sdxl_ip_mask m[SDXL_MAX_IMAGE_PROMPTS];
  static float plane[2 * 16 * 24];
  memset(p, 0, sizeof p);
  memset(m, 0, sizeof m);
  p[0].n_batch = 1; p[0].n_images = 2; p[0].scale = 1.0f; p[0].on_host = 1;
  m[0].mask = plane; m[0].on_host = 1; m[0].height = 16; m[0].width = 24;
  if (SDXL_MAX_IMAGE_PROMPTS != 4 || SDXL_MAX_IP_SOURCES != 8) return 2;
  if (set(NULL, 1, p, m) == 0 || set(NULL, 0, NULL, NULL) == 0) return 3;
  if (offsetof(sdxl_ip_mask, on_host) != sizeof(const float*)) return 4;
  if (offsetof(sdxl_ip_mask, width) != offsetof(sdxl_ip_mask, height) + sizeof(int32_t)) return 5;
  printf("ip_multi_abi_check ok %zu\n", sizeof(sdxl_ip_mask));
  return 0;
}
