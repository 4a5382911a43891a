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
// mu [N,A]; workspace policy_workspace_floats(O, A, H, N) floats.
int policy_step(int O, int A, int H, const float* const params[4], const float* obs, const float* state_in,
                float* state_out, float* mu, int N, float* workspace, cudaStream_t stream);

}  // namespace r2d2
