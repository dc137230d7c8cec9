// Noise schedules and sampler coefficients (DESIGN.md §16). Pure host, float64, no CUDA: the sigma table of an
// alphas_cumprod array, the timestep spacings, and the ONE function that knows which sampler runs — step_coef(), which
// turns (sampler, k, schedule) into the four coefficients of the guided step kernel (kernels.h: guided_step_launch).
// Included by engine.cu (sdxl_schedule_build, sdxl_sample_latent_scheduled) and by testing.cu (sdxl_test_step_coef).
#pragma once
#include "../../include/sdxl_b200.h"

#include <math.h>
#include <stdio.h>

#include <algorithm>
#include <string>
#include <vector>

namespace sdxl {

// log sigma_i of the training timesteps, sigma_i = sqrt((1 - a_i) / a_i)
struct SigmaTable {
  std::vector<double> ls;
  SigmaTable(const double* alphas, int n) : ls(n) {
    for (int i = 0; i < n; ++i) ls[i] = 0.5 * log((1.0 - alphas[i]) / alphas[i]);
  }
  int N() const { return (int)ls.size(); }
  // log sigma is linear in t between floor(t) and ceil(t)
  double sigma(double t) const {
    const int last = N() - 1;
    t = std::min(std::max(t, 0.0), (double)last);
    const int lo = std::min((int)floor(t), std::max(last - 1, 0));
    if (last == 0) return exp(ls[0]);
    const double w = t - lo;
    return exp((1.0 - w) * ls[lo] + w * ls[lo + 1]);
  }
  // the inverse (k-diffusion's sigma_to_t): clamped to [0, N - 1]
  double t_of(double sigma) const {
    const int last = N() - 1;
    if (last == 0) return 0.0;
    const double x = log(sigma);
    int lo = (int)(std::upper_bound(ls.begin(), ls.end(), x) - ls.begin()) - 1;   // largest i with ls[i] <= x
    lo = std::min(std::max(lo, 0), last - 1);
    const double w = std::min(std::max((x - ls[lo]) / (ls[lo + 1] - ls[lo]), 0.0), 1.0);
    return lo + w;
  }
};

// Empty when `s` is a schedule this library can build over n_train timesteps, else the reason, naming the field.
inline std::string schedule_problem(const sdxl_schedule* s, int n_train) {
  char b[256];
  b[0] = 0;
  const int N = n_train;
  if (!s) return "schedule: null";
  if (s->sampler < 0 || s->sampler > SDXL_SAMPLER_LCM) snprintf(b, sizeof b, "schedule: sampler = %d outside [0, %d]", s->sampler, SDXL_SAMPLER_LCM);
  else if (s->spacing < 0 || s->spacing > SDXL_SPACING_LCM) snprintf(b, sizeof b, "schedule: spacing = %d outside [0, %d]", s->spacing, SDXL_SPACING_LCM);
  else if (s->n_steps < 1 || s->n_steps > N) snprintf(b, sizeof b, "schedule: n_steps = %d outside [1, %d]", s->n_steps, N);
  else if (s->spacing == SDXL_SPACING_LEADING && (s->n_steps - 1) * (N / s->n_steps) + 1 > N - 1)
    snprintf(b, sizeof b, "schedule: n_steps = %d with leading spacing starts at timestep %d, past the last one (%d)", s->n_steps,
             (s->n_steps - 1) * (N / s->n_steps) + 1, N - 1);
  else if (s->spacing == SDXL_SPACING_LCM && (N < 50 || s->n_steps > 50))
    snprintf(b, sizeof b, "schedule: n_steps = %d with LCM spacing must be <= 50 (of %d >= 50 training timesteps)", s->n_steps, N);
  else if (s->first_step < 0 || s->first_step >= s->n_steps) snprintf(b, sizeof b, "schedule: first_step = %d outside [0, %d)", s->first_step, s->n_steps);
  else if (s->last_step < 0 || s->last_step > s->n_steps) snprintf(b, sizeof b, "schedule: last_step = %d outside [0, %d]", s->last_step, s->n_steps);
  else if (s->last_step && s->first_step >= s->last_step) snprintf(b, sizeof b, "schedule: first_step = %d must be below last_step = %d", s->first_step, s->last_step);
  else if (s->renoise != 0 && s->renoise != 1) snprintf(b, sizeof b, "schedule: renoise = %d must be 0 or 1", s->renoise);
  else if (s->renoise && !s->first_step) snprintf(b, sizeof b, "schedule: renoise = 1 needs first_step > 0");
  else if (s->no_cfg != 0 && s->no_cfg != 1) snprintf(b, sizeof b, "schedule: no_cfg = %d must be 0 or 1", s->no_cfg);
  else if (!(s->karras_rho >= 0.f) || !isfinite(s->karras_rho)) snprintf(b, sizeof b, "schedule: karras_rho = %g must be finite and >= 0", s->karras_rho);
  else if (!(s->eta >= 0.f) || !isfinite(s->eta)) snprintf(b, sizeof b, "schedule: eta = %g must be finite and >= 0", s->eta);
  else if (!(s->s_noise >= 0.f) || !isfinite(s->s_noise)) snprintf(b, sizeof b, "schedule: s_noise = %g must be finite and >= 0", s->s_noise);
  return b;
}

// timesteps[0..n) and sigmas[0..n] (sigmas[n] = 0) of a schedule that passed schedule_problem
inline void schedule_fill(const SigmaTable& T, const sdxl_schedule& s, double* t, double* sig) {
  const int N = T.N(), n = s.n_steps;
  for (int k = 0; k < n; ++k) {
    switch (s.spacing) {
      case SDXL_SPACING_REFERENCE: t[k] = N - 1 - k * (N / n); break;
      case SDXL_SPACING_LEADING: t[k] = (n - 1 - k) * (N / n) + 1; break;
      case SDXL_SPACING_TRAILING: t[k] = nearbyint(N - k * ((double)N / n)) - 1; break;   // ties to even, as numpy rounds
      case SDXL_SPACING_LINSPACE: t[k] = n == 1 ? N - 1 : (N - 1) * (1.0 - (double)k / (n - 1)); break;
      case SDXL_SPACING_KARRAS: {
        const double rho = s.karras_rho > 0.f ? s.karras_rho : 7.0;
        const double a = pow(exp(T.ls[N - 1]), 1.0 / rho), b = pow(exp(T.ls[0]), 1.0 / rho);
        sig[k] = pow(a + (n == 1 ? 0.0 : (double)k / (n - 1)) * (b - a), rho);
        t[k] = T.t_of(sig[k]);
        continue;
      }
      default: {   // SDXL_SPACING_LCM: diffusers' LCMScheduler.set_timesteps, original_inference_steps = 50
        const int j = (int)floor(k * (50.0 / n));   // floor(linspace(0, 50, n, endpoint = False))[k]
        t[k] = (50 - j) * (N / 50) - 1;
      }
    }
    sig[k] = T.sigma(t[k]);
  }
  sig[n] = 0.0;
}

// The sampler layer. Step k of the schedule takes the state xh at sigma_k to sigma_{k+1}:
//   xh' = cx * xh + cd * D + ch * D_prev + cn * z,   D = xh - sigma_k * eps (d_scale),   x_in' = c_in * xh'
// `has_prev`: D of step k - 1 is in the history buffer (false on the first step of a call).
// The denoised latent D = dx * xh - de * g of the model output g at sigma (DESIGN.md §18), in double: an epsilon model gives
// D = xh - sigma * eps (the step kernel's own expression, dx = 1, de = sigma), a v model D = xh / (sigma^2 + 1) - sigma / sqrt(sigma^2 + 1) * v.
struct DScale {
  float dx, de;
};
inline DScale d_scale(int prediction, double sigma) {
  if (prediction != SDXL_PREDICTION_V) return {1.f, (float)sigma};
  return {(float)(1.0 / (sigma * sigma + 1.0)), (float)(sigma / sqrt(sigma * sigma + 1.0))};
}
struct StepCoef {
  float cx, cd, ch, cn, c_in;
};
inline bool sampler_keeps_history(int sampler) { return sampler == SDXL_SAMPLER_DPMPP_2M; }
inline StepCoef step_coef(const sdxl_schedule& s, int k, const double* t, const double* sig, bool has_prev) {
  const double sg = sig[k], sn = sig[k + 1];
  double cx = 0, cd = 0, ch = 0, cn = 0;
  switch (s.sampler) {
    case SDXL_SAMPLER_EULER:
      cx = sn / sg;
      cd = 1.0 - cx;
      break;
    case SDXL_SAMPLER_EULER_ANCESTRAL: {
      const double eta = s.eta > 0.f ? s.eta : 1.0, s_noise = s.s_noise > 0.f ? s.s_noise : 1.0;
      const double su = std::min(sn, eta * sqrt(sn * sn * (sg * sg - sn * sn) / (sg * sg)));
      const double sd = sqrt(sn * sn - su * su);
      cx = sd / sg;
      cd = 1.0 - cx;
      cn = s_noise * su;
      break;
    }
    case SDXL_SAMPLER_DPMPP_2M: {
      cx = sn / sg;
      if (sn == 0.0) {   // h = inf: E = 1, first order
        cd = 1.0;
        break;
      }
      const double h = log(sg / sn), E = -expm1(-h);
      if (!has_prev || k == 0) {
        cd = E;
        break;
      }
      const double r = log(sig[k - 1] / sg) / h;
      cd = E * (1.0 + 1.0 / (2.0 * r));
      ch = -E / (2.0 * r);
      break;
    }
    default: {   // SDXL_SAMPLER_LCM: boundary-condition scalings with timestep scaling 10 and sigma_data 0.5
      const double ts = 10.0 * t[k];
      cx = 0.25 / (ts * ts + 0.25) / sqrt(sg * sg + 1.0);
      cd = ts / sqrt(ts * ts + 0.25);
      cn = sn;
    }
  }
  return {(float)cx, (float)cd, (float)ch, (float)cn, (float)(1.0 / sqrt(sn * sn + 1.0))};
}

}  // namespace sdxl
