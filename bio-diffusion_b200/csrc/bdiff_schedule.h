// bdiff_schedule.h — the host half of bdiff_sample and bdiff_inpaint: the noise schedule's tables, the RePaint program,
// the centring of the inpainted molecules and the argument checks.  Plain C++17
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

// The RePaint program of inpaint, unrolled (bdiff/schedule.py repaint_schedule / repaint_program).  Every denoise op moves
// z from t = s+1 to s; the last op of every segment but the final one is followed by a jump back from s to t = s + j.
// Draws (include/bdiff.h): z_T takes 0 and 1; then in chain order each op takes 4 (known x, known h, unknown x, unknown h)
// and each jump 2 (x, h); the decode takes the last 2.
struct RepaintProgram {
  std::vector<int32_t> sched;          // denoising ops of each segment (get_repaint_schedule)
  std::vector<int32_t> op_s;           // [ops] grid point s each op lands on
  std::vector<uint8_t> jump_after;     // [ops] 1: a jump back follows the op
  std::vector<int32_t> slot;           // [ops] frame slot of the op; return_frames = the dummy slot (no frame)
  std::vector<float> rev;              // [ops * 4] {alpha_ts, c_eps, sigma, t}: rows of schedule_tables
  std::vector<float> known;            // [ops * 2] {alpha_s, sigma_s}
  std::vector<float> jump;             // [jumps * 4] {alpha_t|s, sigma_t|s, s, t}
  std::vector<uint64_t> op_draw;       // [ops] the op's first draw (known x)
  std::vector<uint64_t> jump_draw;     // [jumps] the jump's first draw (x)
  uint64_t decode_draw = 0;            // the decode's first draw
  float dec[4] = {0.f, 0.f, 0.f, 0.f}; // the decode row of schedule_tables
};

// Why a chain of num_timesteps steps cannot return `return_frames` frames ("" = it can): schedule.py check_frames.
inline std::string frames_args_error(int num_timesteps, int return_frames) {
  char buf[160];
  if (!(0 < return_frames && return_frames <= num_timesteps)) {
    snprintf(buf, sizeof buf, "return_frames must be in [1, num_timesteps=%d], got %d", num_timesteps, return_frames);
    return buf;
  }
  if (num_timesteps % return_frames) {
    snprintf(buf, sizeof buf, "return_frames=%d does not divide num_timesteps=%d", return_frames, num_timesteps);
    return buf;
  }
  return "";
}

// Why a RePaint program cannot be built ("" = it can): check_repaint of schedule.py.
inline std::string repaint_args_error(int num_timesteps, int resamplings, int jump_length, int return_frames) {
  if (resamplings < 1 || jump_length < 1 || num_timesteps < 1) {
    char buf[160];
    snprintf(buf, sizeof buf, "num_resamplings, jump_length and num_timesteps must be >= 1 (got %d, %d, %d)", resamplings,
             jump_length, num_timesteps);
    return buf;
  }
  const std::string why = frames_args_error(num_timesteps, return_frames);
  if (!why.empty()) return why;
  if (jump_length > 1 && return_frames > 1) return "chain visualisation (return_frames > 1) is only defined for jump_length == 1";
  return "";
}

// Frame slot written after the step that lands on s (schedule.py frame_slot), or -1.
inline int frame_slot(long long s, long long num_timesteps, long long return_frames) {
  return (s * return_frames) % num_timesteps == 0 ? (int)(s * return_frames / num_timesteps) : -1;
}

// The program for arguments repaint_args_error accepts.  Reverse rows are gathered from schedule_tables(gamma, T), so an
// op is bit-identical to bdiff_sample's step at the same s; the known and jump rows are evaluated in fp64 at the fp32 grid
// and gamma values like schedule_tables' and rounded once.
inline RepaintProgram repaint_program(const std::vector<float>& gamma, int resamplings, int jump_length, int num_timesteps,
                                      int return_frames) {
  RepaintProgram g;
  const int T = num_timesteps, J = jump_length, TM = (int)gamma.size() - 1;
  for (int curr = 0; curr < T;) {                        // get_repaint_schedule, built back to front
    if (curr + J < T) {
      if (!g.sched.empty()) g.sched.back() += J;
      g.sched.insert(g.sched.end(), g.sched.empty() ? resamplings : resamplings - 1, J);
      curr += J;
    } else {
      if (!g.sched.empty()) g.sched.back() += T - curr;
      else g.sched.push_back(T - curr);
      curr = T;
    }
  }
  std::vector<int32_t> sched(g.sched.rbegin(), g.sched.rend());
  g.sched = sched;
  std::vector<float> coef((size_t)T * 4);
  schedule_tables(gamma, T, coef.data(), g.dec);
  auto gam = [&](float v) { return (double)gamma[(size_t)nearbyintf(v * (float)TM)]; };
  uint64_t draw = 2;
  int s = T - 1;
  for (size_t i = 0; i < sched.size(); ++i) {
    const bool last_seg = i + 1 == sched.size();
    for (int jj = 0; jj < sched[i]; ++jj) {
      g.op_s.push_back(s);
      const int slot = sched[i] > J || last_seg ? frame_slot(s, T, return_frames) : -1;
      g.slot.push_back(slot < 0 ? return_frames : slot);
      g.rev.insert(g.rev.end(), coef.begin() + 4 * (size_t)(T - 1 - s), coef.begin() + 4 * (size_t)(T - s));
      const double g_s = gam((float)s / (float)T);
      g.known.push_back((float)std::sqrt(d_sigmoid(-g_s)));
      g.known.push_back((float)std::sqrt(d_sigmoid(g_s)));
      g.op_draw.push_back(draw);
      draw += 4;
      const bool jump = jj == sched[i] - 1 && !last_seg;
      g.jump_after.push_back(jump ? 1 : 0);
      if (jump) {
        const float js = (float)s / (float)T, jt = (float)(s + J) / (float)T;
        const double a_s = gam(js), a_t = gam(jt);
        const double sigma2_ts = -std::expm1(d_softplus(a_s) - d_softplus(a_t));
        g.jump.push_back((float)std::exp(0.5 * (d_logsigmoid(-a_t) - d_logsigmoid(-a_s))));
        g.jump.push_back((float)std::sqrt(sigma2_ts));
        g.jump.push_back(js);
        g.jump.push_back(jt);
        g.jump_draw.push_back(draw);
        draw += 2;
        s += J;
      }
      --s;
    }
  }
  g.decode_draw = draw;
  return g;
}

// xh0[:, :3] -= the mean position of the molecule's fixed atoms (GCDMSampler.inpaint): sequential fp32 sums of x * fixed
// over the molecule's atoms in order, the count of fixed atoms, and the mean tot / max(count, 1), so a molecule without
// fixed atoms is not moved.  xh0 is [N, ld] row-major.
inline void center_on_fixed(int num_mols, const int32_t* num_nodes, int ld, const uint8_t* fixed, float* xh0) {
  for (int k = 0, i0 = 0; k < num_mols; i0 += num_nodes[k++]) {
    float tot[3] = {0.f, 0.f, 0.f}, cnt = 0.f;
    for (int i = i0; i < i0 + num_nodes[k]; ++i) {
      const float f = fixed[i] ? 1.f : 0.f;
      for (int c = 0; c < 3; ++c) tot[c] += xh0[(size_t)i * ld + c] * f;
      cnt += f;
    }
    const float div = std::fmax(cnt, 1.f);
    const float mean[3] = {tot[0] / div, tot[1] / div, tot[2] / div};
    for (int i = i0; i < i0 + num_nodes[k]; ++i)
      for (int c = 0; c < 3; ++c) xh0[(size_t)i * ld + c] -= mean[c];
  }
}

// Why bdiff_inpaint refuses its arguments ("" = accepted).
inline std::string inpaint_args_error(int num_h, int num_context, const bdiff_sample_config& c, int num_mols,
                                      const int32_t* num_nodes_host, const float* context, int num_timesteps,
                                      int resamplings, int jump_length, int return_frames, const float* xh0_host,
                                      const uint8_t* fixed_host, const float* out) {
  std::string why = sample_args_error(num_h, num_context, c, num_mols, num_nodes_host, context, num_timesteps, nullptr,
                                      nullptr, out);
  if (!why.empty()) return why;
  why = repaint_args_error(num_timesteps, resamplings, jump_length, return_frames);
  if (!why.empty()) return why;
  if (!xh0_host) return "xh0_host is NULL";
  if (!fixed_host) return "fixed_host is NULL";
  long long n = 0;
  for (int k = 0; k < num_mols; ++k) n += num_nodes_host[k];
  for (long long i = 0; i < n; ++i)
    if (fixed_host[i] > 1) {
      char buf[96];
      snprintf(buf, sizeof buf, "fixed_host[%lld] = %d: must be 0 or 1", i, (int)fixed_host[i]);
      return buf;
    }
  return "";
}

}  // namespace bdiff
