// TEST INFRASTRUCTURE: the host (g++) build of the step kernel's logic (env_harness.cpp) with the robot's own policy
// (cn_config.robot_policy 1 'orca' / 2 'social_force', cn_robot_act in cn_env_core.cuh).  The step loop is the one of
// env_harness.cpp: its cn_phase_load runs the robot's policy once robot_policy is set.  This file adds the robot's
// parameter and state (fp64 velocity, frozen rvo2 simulator) to a harness created there.
#include "env_harness.cpp"

extern "C" void* robot_harness_create(const cn_config* cfg) {
  Harness* hn = static_cast<Harness*>(harness_create(cfg));
  hn->p.robot_policy = cfg->robot_policy;
  const size_t N = hn->p.N, NH = N * hn->p.H;
  CnState& g = hn->g;
  halloc(hn, "rwx", &g.rwx, N); halloc(hn, "rwy", &g.rwy, N);
  halloc(hn, "rsim_exists", &g.rsim_exists, N); halloc(hn, "rsim_nd", &g.rsim_nd, N);
  halloc(hn, "rsim_rother", &g.rsim_rother, NH);
  return hn;
}
