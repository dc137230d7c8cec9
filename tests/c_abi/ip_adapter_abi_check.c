/* Plain-C consumer of the IP-Adapter and CLIP vision entry points of include/sdxl_b200.h: they link against libsdxl_b200.so with the
 * prototypes of the header, and NULL objects are refused without touching a GPU. Built and run by tests/test_ip_adapter_cpu.py. */
#include <stddef.h>
#include <stdio.h>

#include "sdxl_b200.h"

int main(void) {
  int (*load)(sdxl_ctx*, const sdxl_ip_adapter_cfg*, const void*, size_t, int, sdxl_ip_adapter**) = sdxl_ip_adapter_load;
  void (*destroy)(sdxl_ip_adapter*) = sdxl_ip_adapter_destroy;
  int (*set)(sdxl_unet*, const sdxl_image_prompt*) = sdxl_unet_set_image_prompt;
  int (*project)(sdxl_ip_adapter*, int, const float*, int, sdxl_half*) = sdxl_ip_adapter_project;
  int (*attn)(sdxl_ctx*, const sdxl_half*, const sdxl_half*, const sdxl_half*, const sdxl_half*, const sdxl_half*, int, int, int, int,
              int, int, float, sdxl_half*) = sdxl_op_ip_attention;
  int (*vload)(sdxl_ctx*, const sdxl_clip_vision_cfg*, const void*, size_t, int, sdxl_clip_vision**) = sdxl_clip_vision_load;
  void (*vdestroy)(sdxl_clip_vision*) = sdxl_clip_vision_destroy;
  int (*encode)(sdxl_clip_vision*, int, const float*, int, float*) = sdxl_clip_vision_encode;
  sdxl_clip_vision* v = NULL;
  sdxl_ip_adapter* a = NULL;
  sdxl_image_prompt p;
  p.adapter = NULL; p.embeds = NULL; p.negative_embeds = NULL; p.on_host = 1; p.n_batch = 1; p.n_images = 1; p.scale = 1.0f;
  p.block_scales_host = NULL;
  if (load(NULL, NULL, NULL, 0, 0, &a) == 0 || set(NULL, &p) == 0 || set(NULL, NULL) == 0 || project(NULL, 1, NULL, 1, NULL) == 0 ||
      attn(NULL, NULL, NULL, NULL, NULL, NULL, 1, 1, 1, 1, 64, 1, 1.0f, NULL) == 0)
    return 3;
  if (vload(NULL, NULL, NULL, 0, 0, &v) == 0 || encode(NULL, 1, NULL, 1, NULL) == 0) return 6;
  vdestroy(NULL);
  destroy(NULL);
  if (offsetof(sdxl_ip_adapter_cfg, image_embed_dim) != sizeof(sdxl_unet_cfg)) return 4;
  printf("ip_adapter_abi_check ok %zu %zu %zu\n", sizeof(sdxl_clip_vision_cfg), sizeof(sdxl_image_prompt), sizeof(sdxl_ip_adapter_cfg));
  return 0;
}
