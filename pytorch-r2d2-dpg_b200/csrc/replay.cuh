#pragma once
#include "common.cuh"

namespace r2d2 {

constexpr int TREE_K = 32;          // fan-out: one 128-byte line of fp32 partial sums per node
constexpr int TREE_MAX_LEVELS = 8;  // 32^7 leaves is far beyond 180 GB of rows

struct TreeView {
  float* lvl[TREE_MAX_LEVELS];      // lvl[0] = leaf priorities (one per row), lvl[levels-1][0] = total
  long long n[TREE_MAX_LEVELS];
  int levels;
};

struct Replay;
int replay_create(Replay** out, const r2d2_replay_config* cfg);
int replay_destroy(Replay* r);
int replay_set_priority_exponent(Replay* r, float alpha);
int replay_add_episode(Replay* r, const float* obs, const float* act, const float* rew, const float* term,
                       const float* states, int n_rows, int n_state_rows, const float* priority, int n_starts,
                       cudaStream_t stream);
int replay_add_episodes(Replay* r, int n_episodes, const int* n_rows, const int* n_starts, const float* obs,
                        const float* act, const float* rew, const float* term, const float* states,
                        const float* leaf_prio, long long* row_start_out, long long* n_evicted_out,
                        long long* sequence_counter_out, cudaStream_t stream);
int replay_sample(Replay* r, const float* u, int batch, long long* leaf_idx, float* obs, float* act, float* rew,
                  float* term, float* states, cudaStream_t stream);
int replay_sample_weighted(Replay* r, const float* u, int batch, float beta, long long* leaf_idx, float* is_weight,
                           float* obs, float* act, float* rew, float* term, float* states, cudaStream_t stream);
int replay_gather(Replay* r, const long long* leaf_idx, int batch, float* obs, float* act, float* rew, float* term,
                  float* states, cudaStream_t stream);
int replay_update_priorities(Replay* r, const long long* leaf_idx, const float* prio, int batch, cudaStream_t stream);
int replay_stats(Replay* r, r2d2_replay_stats_t* out, cudaStream_t stream);
int replay_decode(Replay* r, const long long* leaf_host, int n, long long* episode_index, long long* sequence_index);
int replay_tree_level(Replay* r, int level, const float** dev_ptr, long long* n);

}  // namespace r2d2
