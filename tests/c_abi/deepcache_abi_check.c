/* Plain-C consumer of the DeepCache entry point of include/sdxl_b200.h: it links against libsdxl_b200.so with the prototype of the
 * header, and a NULL UNet is refused without touching a GPU. Built and run by tests/test_deepcache_cpu.py. */
#include <stddef.h>
#include <stdio.h>

#include "sdxl_b200.h"

int main(void) {
  int (*set)(sdxl_unet*, const sdxl_deepcache*) = sdxl_unet_set_deepcache;
  sdxl_deepcache d;
  d.interval = 3; d.branch = 0; d.forward_cached = 0;
  if (set(NULL, &d) == 0 || set(NULL, NULL) == 0) return 3;
  if (offsetof(sdxl_deepcache, branch) != 4 || offsetof(sdxl_deepcache, forward_cached) != 8) return 4;
  printf("deepcache_abi_check ok %zu\n", sizeof(sdxl_deepcache));
  return 0;
}
