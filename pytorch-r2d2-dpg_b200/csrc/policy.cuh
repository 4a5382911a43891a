// One env step of the four recurrent nets of many actor lanes (Actor.run, actor.py:149-154), fp32 FMA on the flat
// state_dict blocks.  Five launches chained with programmatic dependent launch; see policy.cu.
#pragma once
#include "common.cuh"

namespace r2d2 {

constexpr int kPolicyMaxLanes = 256;
constexpr int kPolicyMaxHidden = 512;
constexpr int kPolicyMaxActions = 64;

// floats of workspace one step needs for N lanes
size_t policy_workspace_floats(int O, int A, int H, int N);

// params[4]: actor, target_actor, critic, target_critic.  obs [N,O]; state_in / state_out [4,2,N,H] (must not alias);
// mu [N,A]; workspace policy_workspace_floats(O, A, H, N) floats.  obs_mean / obs_inv_std [O] (both or neither):
// phase 1 reads obs_norm_apply(obs) instead of obs (r2d2_policy_step_ex).
// explore (r2d2_policy_step_explore): the head phase also writes action [N,A] = clip(mu + noise) with the lanes' noise
// (r2d2_exploration, checked here: sigma is read back, which synchronises the stream); nullptr is the plain step.
int policy_step(int O, int A, int H, const float* const params[4], const float* obs, const float* state_in,
                float* state_out, float* mu, int N, float* workspace, cudaStream_t stream,
                const float* obs_mean = nullptr, const float* obs_inv_std = nullptr, float obs_clip = 0.f,
                const r2d2_exploration* explore = nullptr, float* action = nullptr);

}  // namespace r2d2
