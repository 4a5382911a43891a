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

// Global sampling over the replay shards of W data-parallel ranks (include/r2d2_b200.h, r2d2_replay_attach_group).
// Every rank owns one buffer of `GlobalLayout::bytes` that every rank maps: an exchange block
//   [ flags 256 B | totals [16] | minima [16] | own min | uniforms [W*B] | records: leaf [W*B], shard [W*B], prio [W*B]
//     | drawn leaf per global draw (-1: another shard's) [W*B] ]
// and the rank's two batch slots (obs, act, rew, term, states, leaf_idx, shard, is_weight, uniforms), which the owners
// of the drawn rows write with peer stores.  Global draw j = c*B + b is trained by rank c in column b.
constexpr int kGlobalMaxWorld = 16;
constexpr int kGlobalFlagPub = 0, kGlobalFlagTot = 16, kGlobalFlagDel = 32, kGlobalStatus = 48;   // uint32 words
constexpr size_t kGlobalOffTotals = 256, kGlobalOffMinima = 320, kGlobalOffOwnMin = 384;

struct GlobalLayout {
  size_t bytes = 0, exchange_bytes = 0, slot_bytes = 0;
  size_t off_uniforms = 0, off_rec_leaf = 0, off_rec_shard = 0, off_rec_prio = 0, off_draw_leaf = 0;   // exchange
  size_t off_obs = 0, off_act = 0, off_rew = 0, off_term = 0, off_states = 0, off_leaf = 0, off_shard = 0,
         off_weight = 0, off_slot_uniforms = 0;                                                        // in a slot
  __host__ __device__ size_t slot(int s) const { return exchange_bytes + (size_t)s * slot_bytes; }
};
GlobalLayout global_layout(int T, int B, int O, int A, int H, int world);

struct GlobalPeers { char* base[kGlobalMaxWorld]; };

// exchange kernels (global_replay.cu)
int global_publish_records(const GlobalPeers& p, const GlobalLayout& lay, int world, int rank, int B,
                           const long long* leaf, const int* shard, const float* prio, unsigned epoch, cudaStream_t st);
int global_publish_root(const GlobalPeers& p, const GlobalLayout& lay, int world, int rank, int B, int slot,
                        const float* root, unsigned epoch, cudaStream_t st);
int global_deliver(const GlobalPeers& p, int world, int rank, unsigned epoch, cudaStream_t st);
int global_receive(const GlobalPeers& p, const GlobalLayout& lay, int world, int rank, int B, int slot, bool weighted,
                   float beta, unsigned epoch, cudaStream_t st);

struct Replay;
int replay_create(Replay** out, const r2d2_replay_config* cfg, const r2d2_replay_options* options);   // null: defaults
int replay_device_bytes(Replay* r, size_t* out);
int replay_host_bytes(Replay* r, size_t* out);
int replay_destroy(Replay* r);
int replay_set_priority_exponent(Replay* r, float alpha);
int replay_add_episode(Replay* r, const float* obs, const float* act, const float* rew, const float* term,
                       const float* states, int n_rows, int n_state_rows, const float* priority, int n_starts,
                       cudaStream_t stream);
int replay_add_episodes(Replay* r, int n_episodes, const int* n_rows, const int* n_starts, const float* obs,
                        const float* act, const float* rew, const float* term, const float* states,
                        const float* leaf_prio, long long* row_start_out, long long* n_evicted_out,
                        long long* sequence_counter_out, cudaStream_t stream, double* obs_moments = nullptr,
                        long long* n_nonfinite_out = nullptr);
int replay_set_obs_normalizer(Replay* r, const float* mean_f, const float* inv_std_f, float clip);
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
int replay_export_info(Replay* r, r2d2_replay_snapshot_info* out);
int replay_export_episodes(Replay* r, long long* row_start, int* n_rows, int* n_starts, long long* serial);
int replay_export_rows(Replay* r, long long first, long long n, float* obs, float* act, float* rew, float* term,
                       void* states, float* leaves, cudaStream_t stream);
int replay_import_begin(Replay* r, const r2d2_replay_snapshot_info* info, const long long* row_start,
                        const int* n_rows, const int* n_starts, const long long* serial, long long* n_dropped_out,
                        cudaStream_t stream);
int replay_import_rows(Replay* r, long long first, long long n, const float* obs, const float* act, const float* rew,
                       const float* term, const void* states, const float* leaves, cudaStream_t stream);
int replay_import_end(Replay* r, cudaStream_t stream);
int replay_attach_group(Replay* r, int rank, int world, int batch, void* const* peer_bases, size_t buffer_bytes);
int replay_global_write_back(Replay* r, int stage, const long long* leaf, const int* shard, const float* prio,
                             cudaStream_t stream);
int replay_global_draw(Replay* r, int stage, int slot, int weighted, float beta, cudaStream_t stream);
int replay_global_status(Replay* r, int* out, cudaStream_t stream);

}  // namespace r2d2
