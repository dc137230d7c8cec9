/* Plain-C consumer of the DPM++ 2M SDE, DPM++ 3M SDE, UniPC, Heun and DPM2 sampler values of include/sdxl_b200.h: each builds a
 * schedule on the host without a GPU, the unassigned 4 and the value past the last sampler are refused naming the field, and the
 * values keep their numbers. Built and run by tests/test_samplers2_cpu.py. */
#include <math.h>
#include <stdio.h>
#include <string.h>

#include "sdxl_b200.h"

int main(void) {
  static const int samplers[] = {SDXL_SAMPLER_DPMPP_2M_SDE, SDXL_SAMPLER_DPMPP_3M_SDE, SDXL_SAMPLER_UNIPC, SDXL_SAMPLER_HEUN,
                                 SDXL_SAMPLER_DPM_2};
  double alphas[100], t[8], sig[9], a = 1.0;
  sdxl_schedule s;
  int i;
  if (SDXL_SAMPLER_LCM != 3 || SDXL_SAMPLER_DPMPP_2M_SDE != 5 || SDXL_SAMPLER_DPMPP_3M_SDE != 6 || SDXL_SAMPLER_UNIPC != 7 ||
      SDXL_SAMPLER_HEUN != 8 || SDXL_SAMPLER_DPM_2 != 9)
    return 2;
  for (i = 0; i < 100; ++i) {
    a *= 1.0 - (0.001 + 0.0005 * i);
    alphas[i] = a;
  }
  for (i = 0; i < 5; ++i) {
    memset(&s, 0, sizeof s);
    s.sampler = samplers[i];
    s.spacing = SDXL_SPACING_KARRAS;
    s.n_steps = 8;
    s.eta = 0.5f;
    if (sdxl_schedule_build(alphas, 100, &s, t, sig) != 0) return 3;
    if (sig[8] != 0.0 || !(sig[7] < sig[6])) return 4;
  }
  s.sampler = SDXL_SAMPLER_DPM_2 + 1;
  if (sdxl_schedule_build(alphas, 100, &s, t, sig) == 0 || !strstr(sdxl_schedule_last_error(), "sampler")) return 5;
  s.sampler = 4;
  if (sdxl_schedule_build(alphas, 100, &s, t, sig) == 0 || !strstr(sdxl_schedule_last_error(), "sampler")) return 6;
  printf("sampler2_abi_check ok %d\n", SDXL_SAMPLER_DPM_2);
  return 0;
}
