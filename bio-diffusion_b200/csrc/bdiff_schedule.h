// bdiff_schedule.h — the host half of bdiff_sample: the noise schedule's tables and the argument checks.  Plain C++17
// without CUDA headers, so that the CPU suite compiles it with g++ (tests/native/sample_hostcheck.cpp).
//
// The tables restate bdiff/schedule.py (gamma_table, step_coefficient_table, decode_coefficients).  gamma is fp64 exactly
// as numpy builds it (bit-equal after the rounding to fp32); the coefficients are evaluated in fp64 and rounded once,
// so they do not depend on a vector math library.  schedule.py evaluates them in fp32 with torch's CPU kernels, whose
// rounding errors the cancellation in sigma2_ts = -expm1(softplus(g_s) - softplus(g_t)) magnifies: its c_eps and sigma
// can differ from these in the last few digits (tests/test_native_sample_cpu.py bounds by how much).  Built with
// -ffp-contract=off so that the gamma recurrence rounds where numpy does.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/bdiff.h"

namespace bdiff {

// gamma[0..T] of PredefinedNoiseSchedule (variational_diffusion.py:68-107): polynomial schedule + clip_noise_schedule.
inline std::vector<float> schedule_gamma(int T, double power, double precision) {
  const int steps = T + 1;
  // np.linspace(0, steps, steps): i * (steps / (steps - 1)), the last point exactly `steps`
  const double step = (double)steps / (double)(steps - 1);
  std::vector<double> a(steps + 1);
  a[0] = 1.0;
  for (int i = 0; i < steps; ++i) {
    const double x = i == steps - 1 ? (double)steps : (double)i * step;
    const double r = x / steps;
    const double p = power == 2.0 ? r * r : std::pow(r, power);
    const double q = 1.0 - p;
    a[i + 1] = q * q;
  }
  std::vector<float> g(steps);
  double acc = 1.0;
  for (int i = 0; i < steps; ++i) {
    double ratio = a[i + 1] / a[i];
    ratio = std::fmin(std::fmax(ratio, 0.001), 1.0);     // np.clip
    acc *= ratio;                                        // np.cumprod
    const double alpha2 = (1.0 - 2.0 * precision) * acc + precision;
    const double sigma2 = 1.0 - alpha2;
    g[i] = (float)(-(std::log(alpha2) - std::log(sigma2)));
  }
  return g;
}

inline double d_softplus(double x) { return x > 20.0 ? x : std::log1p(std::exp(x)); }
inline double d_logsigmoid(double x) { return std::fmin(0.0, x) - std::log1p(std::exp(-std::fabs(x))); }
inline double d_sigmoid(double x) { return 1.0 / (1.0 + std::exp(-x)); }

// Rows {alpha_ts, c_eps, sigma, t} for s = S-1 .. 0 (transition_terms + _reverse_rows of schedule.py) and the decode row
// {1/alpha_0, sigma_0, sigma_x, 0}.  The grid points and the gamma lookup follow schedule.py in fp32; each coefficient is
// then evaluated in fp64 from the fp32 gamma values and rounded once.
inline void schedule_tables(const std::vector<float>& gamma, int S, float* coef, float* dec) {
  const int T = (int)gamma.size() - 1;
  for (int r = 0; r < S; ++r) {
    const float s_int = (float)(S - 1 - r), t_int = s_int + 1.f;
    const float s = s_int / (float)S, t = t_int / (float)S;
    const double g_s = gamma[(size_t)nearbyintf(s * (float)T)], g_t = gamma[(size_t)nearbyintf(t * (float)T)];
    const double sigma2_ts = -std::expm1(d_softplus(g_s) - d_softplus(g_t));
    const double alpha_ts = std::exp(0.5 * (d_logsigmoid(-g_t) - d_logsigmoid(-g_s)));
    const double sigma_s = std::sqrt(d_sigmoid(g_s)), sigma_t = std::sqrt(d_sigmoid(g_t));
    coef[4 * r + 0] = (float)alpha_ts;
    coef[4 * r + 1] = (float)(sigma2_ts / alpha_ts / sigma_t);
    coef[4 * r + 2] = (float)(std::sqrt(sigma2_ts) * sigma_s / sigma_t);
    coef[4 * r + 3] = t;
  }
  const double g0 = gamma[0];
  dec[0] = (float)(1.0 / std::sqrt(d_sigmoid(-g0)));
  dec[1] = (float)std::sqrt(d_sigmoid(g0));
  dec[2] = (float)std::exp(0.5 * g0);
  dec[3] = 0.f;
}

inline const char* sample_config_error(const bdiff_sample_config& c) {
  if (c.num_atom_types < 1 || (c.include_charges != 0 && c.include_charges != 1)) return "bad num_atom_types / include_charges";
  if (c.model_timesteps < 1) return "model_timesteps must be >= 1";
  if (!(c.schedule_power > 0.0) || !(c.noise_precision > 0.0) || !(c.noise_precision < 0.5))
    return "schedule_power must be > 0 and noise_precision in (0, 0.5)";
  return nullptr;
}

// Why bdiff_sample refuses its arguments ("" = accepted).  num_h / num_context come from the handle's bdiff_config.
inline std::string sample_args_error(int num_h, int num_context, const bdiff_sample_config& c, int num_mols,
                                     const int32_t* num_nodes_host, const float* context, int num_timesteps,
                                     const float* z_init, const int64_t* z_init_shape, const float* xh) {
  char buf[160];
  if (num_h != c.num_atom_types + c.include_charges) return "bdiff_sample_setup: num_atom_types + include_charges != num_h";
  if (num_mols < 1) return "num_mols must be >= 1";
  if (!num_nodes_host) return "num_nodes_host is NULL";
  long long n = 0;
  for (int k = 0; k < num_mols; ++k) {
    if (num_nodes_host[k] < 1) {
      snprintf(buf, sizeof buf, "num_nodes_host[%d] = %d: every molecule needs at least one atom", k, num_nodes_host[k]);
      return buf;
    }
    n += num_nodes_host[k];
  }
  if (n > (1ll << 30)) return "too many atoms";
  if (num_timesteps < 1) return "num_timesteps must be >= 1";
  if (num_context > 0 && !context) {
    snprintf(buf, sizeof buf, "context [num_mols, %d] is required by a property-conditional configuration", num_context);
    return buf;
  }
  if (z_init) {
    if (!z_init_shape) return "z_init given without z_init_shape";
    if (z_init_shape[0] != n || z_init_shape[1] != 3 + num_h) {
      snprintf(buf, sizeof buf, "z_init must be [%lld, %d], got [%lld, %lld]", n, 3 + num_h, (long long)z_init_shape[0],
               (long long)z_init_shape[1]);
      return buf;
    }
  }
  if (!xh) return "xh is NULL";
  return "";
}

}  // namespace bdiff
