// Host build of bdiff_sample's argument checks (csrc/bdiff_schedule.h) for tests/test_native_sample_cpu.py: no CUDA
// runtime, so the checks run on a machine without a GPU.
#include <cstring>

#include "../../bio-diffusion_b200/csrc/bdiff_schedule.h"

extern "C" int sample_hostcheck(int num_h, int num_context, int num_atom_types, int include_charges, int num_mols,
                                const int32_t* num_nodes, int has_context, int num_timesteps, int has_z_init,
                                const int64_t* z_init_shape, char* msg, int msg_bytes) {
  bdiff_sample_config c{};
  c.num_atom_types = num_atom_types;
  c.include_charges = include_charges;
  c.model_timesteps = 1000;
  c.schedule_power = 2.0;
  c.noise_precision = 1e-5;
  static const float dummy = 0.f;
  const std::string why = bdiff::sample_args_error(num_h, num_context, c, num_mols, num_nodes, has_context ? &dummy : nullptr,
                                                   num_timesteps, has_z_init ? &dummy : nullptr, z_init_shape, &dummy);
  std::strncpy(msg, why.c_str(), msg_bytes - 1);
  msg[msg_bytes - 1] = 0;
  return why.empty() ? 0 : BDIFF_EINVAL;
}
