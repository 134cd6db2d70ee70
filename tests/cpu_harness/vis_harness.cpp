// TEST INFRASTRUCTURE: the host (g++) build of the step kernel's logic with robot.visible (cn_config.robot_visible:
// every human's ORCA / social-force solve takes the robot as its last agent, cn_orca_build / cn_sf_action in
// cn_env_core.cuh).  The step loop is the one of env_harness.cpp; the host build of cn_env_core.cuh keeps the
// robot-visible paths and lets the parameter decide, so this file only passes the field through.  It builds on
// robot_harness.cpp so that the ORCA / social-force robot can run among humans that see it.
#include "robot_harness.cpp"

extern "C" void* vis_harness_create(const cn_config* cfg) {
  Harness* hn = static_cast<Harness*>(robot_harness_create(cfg));
  hn->p.robot_visible = cfg->robot_visible;
  return hn;
}
