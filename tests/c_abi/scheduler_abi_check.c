/* Plain-C consumer of the schedule part of include/sdxl_b200.h: it links against libsdxl_b200.so with the prototypes of the header,
 * builds a Karras schedule on the host without touching a GPU, and a NULL UNet is refused. Built and run by
 * tests/test_schedulers_cpu.py. */
#include <math.h>
#include <stddef.h>
#include <stdio.h>
#include <string.h>

#include "sdxl_b200.h"

int main(void) {
  int (*sample)(sdxl_unet*, const sdxl_conditioning*, double, const sdxl_schedule*, const float*, const float*, int, uint64_t,
                const float*, const uint8_t*, float*) = sdxl_sample_latent_scheduled;
  int (*fwd)(sdxl_unet*, int, int, int, const float*, double, float*) = sdxl_unet_forward_f32_at;
  double alphas[100], t[5], sig[6], a = 1.0;
  sdxl_schedule s;
  int i;
  for (i = 0; i < 100; ++i) {
    a *= 1.0 - (0.001 + 0.0005 * i);
    alphas[i] = a;
  }
  memset(&s, 0, sizeof s);
  s.sampler = SDXL_SAMPLER_DPMPP_2M;
  s.spacing = SDXL_SPACING_KARRAS;
  s.n_steps = 5;
  if (sdxl_schedule_build(alphas, 100, &s, t, sig) != 0) return 3;
  if (fabs(sig[0] - sqrt((1.0 - alphas[99]) / alphas[99])) > 1e-12 * sig[0] || sig[5] != 0.0 || fabs(t[0] - 99.0) > 1e-9) return 4;
  for (i = 0; i < 5; ++i)
    if (!(sig[i + 1] < sig[i])) return 5;
  s.n_steps = 101;
  if (sdxl_schedule_build(alphas, 100, &s, t, sig) == 0 || !strstr(sdxl_schedule_last_error(), "n_steps")) return 6;
  if (sample(NULL, NULL, 7.5, &s, NULL, NULL, 0, 0, NULL, NULL, NULL) == 0 || fwd(NULL, 1, 8, 8, NULL, 0.5, NULL) == 0) return 7;
  if (offsetof(sdxl_schedule, n_steps) != 8 || offsetof(sdxl_schedule, no_cfg) != 24 || offsetof(sdxl_schedule, karras_rho) != 28 ||
      offsetof(sdxl_schedule, s_noise) != 36)
    return 8;
  printf("scheduler_abi_check ok %zu\n", sizeof(sdxl_schedule));
  return 0;
}
