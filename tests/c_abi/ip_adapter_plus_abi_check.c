/* Plain-C consumer of the IP-Adapter Plus entry points of include/sdxl_b200.h: they link against libsdxl_b200.so with the prototypes
 * of the header, and NULL objects are refused without touching a GPU. Built and run by tests/test_ip_adapter_plus_cpu.py. */
#include <stddef.h>
#include <stdio.h>
#include <string.h>

#include "sdxl_b200.h"

int main(void) {
  int (*resample)(sdxl_ip_adapter*, int, int, const float*, int, sdxl_half*) = sdxl_ip_adapter_resample;
  int (*hidden)(sdxl_clip_vision*, int, const float*, int, int, float*) = sdxl_clip_vision_encode_hidden;
  int (*set)(sdxl_unet*, const sdxl_image_prompt*) = sdxl_unet_set_image_prompt;
  sdxl_ip_adapter_cfg cfg;
  sdxl_image_prompt p;
  memset(&cfg, 0, sizeof cfg);   /* zero-initialised: resampler_depth = 0 is the base adapter */
  cfg.image_embed_dim = 1280; cfg.tokens_per_image = 16; cfg.resampler_depth = 4; cfg.resampler_heads = 20;
  memset(&p, 0, sizeof p);
  p.n_batch = 1; p.n_images = 1; p.scale = 1.0f; p.seq_len = 257; p.on_host = 1;
  if (resample(NULL, 1, 257, NULL, 1, NULL) == 0 || hidden(NULL, 1, NULL, 1, 31, NULL) == 0 || set(NULL, &p) == 0) return 3;
  if (sdxl_ip_adapter_load(NULL, &cfg, NULL, 0, 0, NULL) == 0) return 5;
  if (offsetof(sdxl_ip_adapter_cfg, image_embed_dim) != sizeof(sdxl_unet_cfg)) return 4;
  if (offsetof(sdxl_ip_adapter_cfg, resampler_depth) != sizeof(sdxl_unet_cfg) + 2 * sizeof(int32_t)) return 6;
  if (offsetof(sdxl_image_prompt, seq_len) <= offsetof(sdxl_image_prompt, block_scales_host)) return 7;
  printf("ip_adapter_plus_abi_check ok %zu %zu\n", sizeof(sdxl_image_prompt), sizeof(sdxl_ip_adapter_cfg));
  return 0;
}
