// Noise schedules and sampler coefficients (DESIGN.md §16, §20). Pure host, float64, no CUDA: the sigma table of an
// alphas_cumprod array, the timestep spacings, and the ONE function that knows which sampler runs — step_stages(), which
// turns (sampler, k, schedule, history) into the one or two evaluations of a step and the coefficient rows of the guided step
// kernel after each (kernels.h: guided_step_launch). Included by engine.cu (sdxl_schedule_build, sdxl_sample_latent_scheduled)
// and by testing.cu (sdxl_test_step_coef, sdxl_test_step_stages).
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
  if (s->sampler < 0 || s->sampler > SDXL_SAMPLER_DPM_2 || (s->sampler > SDXL_SAMPLER_LCM && s->sampler < SDXL_SAMPLER_DPMPP_2M_SDE))
    snprintf(b, sizeof b, "schedule: sampler = %d is not one of [%d, %d] and [%d, %d]", s->sampler, SDXL_SAMPLER_EULER, SDXL_SAMPLER_LCM,
             SDXL_SAMPLER_DPMPP_2M_SDE, SDXL_SAMPLER_DPM_2);
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

// The denoised latent D = dx * xh - de * g of the model output g at sigma (DESIGN.md §18), in double: an epsilon model gives
// D = xh - sigma * eps (the step kernel's own expression, dx = 1, de = sigma), a v model D = xh / (sigma^2 + 1) - sigma / sqrt(sigma^2 + 1) * v.
struct DScale {
  float dx, de;
};
inline DScale d_scale(int prediction, double sigma) {
  if (prediction != SDXL_PREDICTION_V) return {1.f, (float)sigma};
  return {(float)(1.0 / (sigma * sigma + 1.0)), (float)(sigma / sqrt(sigma * sigma + 1.0))};
}
// One evaluation of a step and the launch after it (DESIGN.md §20). The evaluation runs at (t, sigma); then, from the values
// before the launch (the state xh, the saved state xs, the denoised D, the history slots H1 and H2, the noise z):
//   xh' = cx xh + cs xs + cd D + ch H1 + ch2 H2 + cn z                 x_in' = c_in xh'
//   xs' = sx xh + ss xs + sd D + sh H1 + sh2 H2                         (write_xs)
//   H2' = H1 (shift), H1' = D (write_hist)
// D is the evaluation's denoised latent (d_scale above). sigma_next is where the evaluation after this launch runs: the latent
// blend fused into the launch and c_in are at it.
struct Stage {
  double t, sigma, sigma_next;
  float cx, cs, cd, ch, ch2, cn;
  float sx, ss, sd, sh, sh2;
  float c_in;
  bool write_xs, write_hist, shift;
  // the launch reads or writes xs or H2: the step kernel's two-row form (kernels.h: StepRows)
  bool rows() const { return write_xs || shift || cs != 0.f || ch2 != 0.f; }
};
struct StepStages {
  int n;
  Stage st[2];
};
// The sampler layer. Step k of the schedule takes the state xh at sigma_k to sigma_{k+1}. n_hist: the history slots this call
// has filled (min(k - first_step, 2)); multistep history never crosses calls. T: the sigma table, needed only for DPM2's
// midpoint timestep (a null T leaves that stage's t NaN). Every coefficient is computed in double and rounded once.
inline StepStages step_stages(const SigmaTable* T, const sdxl_schedule& s, int k, const double* t, const double* sig, int n_hist) {
  const double sg = sig[k], sn = sig[k + 1];
  StepStages out{};
  out.n = 1;
  Stage& a = out.st[0];
  a.t = t[k];
  a.sigma = sg;
  a.sigma_next = sn;
  double cx = 0, cs = 0, cd = 0, ch = 0, ch2 = 0, cn = 0;
  const double eta = s.eta > 0.f ? s.eta : 1.0, s_noise = s.s_noise > 0.f ? s.s_noise : 1.0;
  const auto fin = [](Stage& q, double x, double xs, double d, double h1, double h2, double z) {
    q.cx = (float)x; q.cs = (float)xs; q.cd = (float)d; q.ch = (float)h1; q.ch2 = (float)h2; q.cn = (float)z;
    q.c_in = (float)(1.0 / sqrt(q.sigma_next * q.sigma_next + 1.0));
  };
  if (s.sampler > SDXL_SAMPLER_LCM && sn == 0.0) {   // the step to sigma = 0 of the new samplers: D exactly, one evaluation
    fin(a, 0, 0, 1, 0, 0, 0);
    return out;
  }
  switch (s.sampler) {
    case SDXL_SAMPLER_DPMPP_2M_SDE: {   // k-diffusion sample_dpmpp_2m_sde, midpoint
      const double h = log(sg / sn), eh = eta * h, phi = -expm1(-h - eh);
      cx = sn / sg * exp(-eh);
      cd = phi;
      if (n_hist >= 1) {
        const double q = 0.5 * phi * h / log(sig[k - 1] / sg);   // 0.5 phi / r, r = h_{k-1} / h
        cd += q;
        ch = -q;
      }
      cn = s_noise * sn * sqrt(-expm1(-2.0 * eh));
      a.write_hist = true;
      fin(a, cx, 0, cd, ch, 0, cn);
      return out;
    }
    case SDXL_SAMPLER_DPMPP_3M_SDE: {   // k-diffusion sample_dpmpp_3m_sde
      const double h = log(sg / sn), he = h * (eta + 1.0), phi1 = -expm1(-he);
      const double phi2 = expm1(-he) / he + 1.0, phi3 = phi2 / he - 0.5;
      double c[3] = {phi1, 0, 0};   // over (D, H1, H2)
      if (n_hist == 1) {
        const double r = log(sig[k - 1] / sg) / h;   // d = (D - H1) / r
        c[0] += phi2 / r;
        c[1] -= phi2 / r;
      } else if (n_hist >= 2) {
        const double r0 = log(sig[k - 1] / sg) / h, r1 = log(sig[k - 2] / sig[k - 1]) / h;
        const double d10[3] = {1.0 / r0, -1.0 / r0, 0.0}, d11[3] = {0.0, 1.0 / r1, -1.0 / r1};
        for (int i = 0; i < 3; ++i) {
          const double d1 = d10[i] + (d10[i] - d11[i]) * r0 / (r0 + r1), d2 = (d10[i] - d11[i]) / (r0 + r1);
          c[i] += phi2 * d1 - phi3 * d2;
        }
      }
      cx = sn / sg * exp(-eta * h);
      cn = s_noise * sn * sqrt(-expm1(-2.0 * eta * h));
      a.write_hist = true;
      a.shift = n_hist >= 1;
      fin(a, cx, 0, c[0], c[1], c[2], cn);
      return out;
    }
    case SDXL_SAMPLER_UNIPC: {   // UniC on the current state (from xs, H1, H2 and D), then UniP from the corrected state
      const int left = s.n_steps - k, order = std::min(std::min(2, n_hist + 1), left);
      double kx = 1, ks = 0, kd = 0, k1 = 0, k2 = 0;   // the corrected state over (xh, xs, D, H1, H2)
      if (n_hist >= 1) {   // corrector of the previous step's predictor order, from sigma_{k-1} to sigma_k
        const double sp = sig[k - 1], hc = log(sp / sg), phc = -expm1(-hc);
        double rho_h = 0.0, rho_d = 0.5;   // order 1: rhos_c = 0.5
        if (n_hist >= 2) {   // order 2: rhos_c = solve([[1, 1], [rk, 1]], [b1, b2]) with bh2's B(h) = expm1(-hc)
          const double rk = -log(sig[k - 2] / sp) / hc, hh = -hc, B = expm1(hh);
          const double hp2 = expm1(hh) / hh - 1.0, hp3 = hp2 / hh - 0.5;
          const double b1 = hp2 / B, b2 = hp3 * 2.0 / B;
          const double rho0 = (b1 - b2) / (1.0 - rk);
          rho_d = b1 - rho0;
          rho_h = rho0 / rk;   // rho0 * (H2 - H1) / rk
        }
        kx = 0;
        ks = sg / sp;
        kd = phc * rho_d;
        k2 = phc * rho_h;
        k1 = phc * (1.0 - rho_h - rho_d);
      }
      const double h = log(sg / sn), phi = -expm1(-h), cr = sn / sg;
      double pd = phi, p1 = 0;
      if (order == 2) {   // rhos_p = 0.5 on D1 = (H1 - D) / r1, r1 = (lambda_{k-1} - lambda_k) / h
        const double r1 = -log(sig[k - 1] / sg) / h;
        pd -= 0.5 * phi / r1;
        p1 += 0.5 * phi / r1;
      }
      a.sx = (float)kx; a.ss = (float)ks; a.sd = (float)kd; a.sh = (float)k1; a.sh2 = (float)k2;
      a.write_xs = true;
      a.write_hist = true;
      a.shift = n_hist >= 1;
      fin(a, cr * kx, cr * ks, cr * kd + pd, cr * k1 + p1, cr * k2, 0);
      return out;
    }
    case SDXL_SAMPLER_HEUN:
    case SDXL_SAMPLER_DPM_2: {   // stage 1: Euler to sigma' (Heun) or sigma_mid (DPM2), saving xh and D
      const bool heun = s.sampler == SDXL_SAMPLER_HEUN;
      const double sm = heun ? sn : exp(0.5 * (log(sg) + log(sn)));
      a.sigma_next = sm;
      a.sx = 1.f;
      a.write_xs = true;
      a.write_hist = heun;
      fin(a, sm / sg, 0, 1.0 - sm / sg, 0, 0, 0);
      Stage& b = out.st[1];
      out.n = 2;
      b.t = heun ? t[k + 1] : (T ? T->t_of(sm) : NAN);
      b.sigma = sm;
      b.sigma_next = sn;
      if (heun)   // x' = xs + (sigma' - sigma) ((xs - H1) / sigma + (xh - D) / sigma') / 2
        fin(b, (sn - sg) / (2.0 * sn), 1.0 + (sn - sg) / (2.0 * sg), -(sn - sg) / (2.0 * sn), -(sn - sg) / (2.0 * sg), 0, 0);
      else   // x' = xs + (sigma' - sigma) (xh - D) / sigma_mid
        fin(b, (sn - sg) / sm, 1.0, -(sn - sg) / sm, 0, 0, 0);
      return out;
    }
    default:
      break;
  }
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
      if (n_hist < 1 || k == 0) {
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
  a.write_hist = s.sampler == SDXL_SAMPLER_DPMPP_2M;
  fin(a, cx, 0, cd, ch, 0, cn);
  return out;
}

}  // namespace sdxl
