// Host build of bdiff_inpaint's centring and argument checks (csrc/bdiff_schedule.h) for
// tests/test_native_inpaint_cpu.py: no CUDA runtime, so they run on a machine without a GPU.
#include <cstring>

#include "../../bio-diffusion_b200/csrc/bdiff_schedule.h"

extern "C" void center_hostcheck(int num_mols, const int32_t* num_nodes, int ld, const uint8_t* fixed, float* xh0) {
  bdiff::center_on_fixed(num_mols, num_nodes, ld, fixed, xh0);
}

extern "C" int inpaint_hostcheck(int num_h, int num_context, int num_atom_types, int include_charges, int num_mols,
                                 const int32_t* num_nodes, int has_context, int num_timesteps, int resamplings,
                                 int jump_length, int return_frames, const uint8_t* fixed, char* msg, int msg_bytes) {
  bdiff_sample_config c{};
  c.num_atom_types = num_atom_types;
  c.include_charges = include_charges;
  c.model_timesteps = 1000;
  c.schedule_power = 2.0;
  c.noise_precision = 1e-5;
  static const float dummy = 0.f;
  const std::string why = bdiff::inpaint_args_error(num_h, num_context, c, num_mols, num_nodes,
                                                    has_context ? &dummy : nullptr, num_timesteps, resamplings,
                                                    jump_length, return_frames, &dummy, fixed, &dummy);
  std::strncpy(msg, why.c_str(), msg_bytes - 1);
  msg[msg_bytes - 1] = 0;
  return why.empty() ? 0 : BDIFF_EINVAL;
}
