// dist.h -- multi-GPU plumbing INSIDE the library (SURVEY.md section 8e): NCCL communicators without torch.
//
// Two ways to get more than one GPU behind the C ABI:
//   * "devices" mode  -- ONE process drives several GPUs: CLIP_B200_DEVICES=0,1,...|all at clip_model_load creates a replica of
//                        the model per device (weights: at most about 5 GB, ViT-bigG/14 f16) and one NCCL communicator per replica (ncclCommInitAll);
//   * "ranks" mode    -- one process per GPU (torchrun / mpirun / any launcher): clip_b200_dist_init(ctx, rank, world, ...) joins
//                        a communicator with ncclCommInitRank; the 128-byte unique id travels through a rendezvous file on the
//                        node (or through the caller's own channel: clip_b200_dist_unique_id + clip_b200_dist_init_with_id).
// The reference's analogue of "several devices inside the library" is ggml-cuda.cu:404-407, 5934-5957 (never compiled by clip.cpp).
// libnccl.so.2 is loaded with dlopen on first use: single-GPU users need no NCCL at all.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <string>

namespace cb {

struct NcclApi;                       // resolved entry points of libnccl.so.2
const NcclApi* nccl_api(std::string& err);      // nullptr + err when the library cannot be loaded

struct DistComm {
    void* comm = nullptr;             // ncclComm_t
    int rank = 0, world = 1;
};

// ---- ranks mode --------------------------------------------------------------------------------------------------------
bool dist_unique_id(void* out128, std::string& err);
// rendezvous == nullptr: derive the path from the launcher's environment (MASTER_PORT + parent pid), see dist.cpp
bool dist_init_rank(DistComm& dc, int rank, int world, const void* id128, std::string& err);
bool dist_rendezvous_id(int rank, int world, const char* rendezvous, void* id128, std::string& err);
void dist_rendezvous_done(int rank);      // rank 0 removes the rendezvous file once the communicator exists
// ---- devices mode ------------------------------------------------------------------------------------------------------
bool dist_init_all(DistComm* comms, const int* devices, int n, std::string& err);
void dist_destroy(DistComm& dc);

// collectives, enqueued on `st` of the CURRENT device (callers in devices mode bracket them with group_start / group_end)
bool dist_all_gather(const DistComm& dc, const void* send, void* recv, size_t bytes_per_rank, cudaStream_t st, std::string& err);
bool dist_all_reduce_max_f64(const DistComm& dc, double* d_buf, size_t n, cudaStream_t st, std::string& err);
bool dist_all_reduce_sum_i32(const DistComm& dc, int32_t* d_buf, size_t n, cudaStream_t st, std::string& err);
bool dist_group_start(std::string& err);
bool dist_group_end(std::string& err);
int dist_nccl_version();

// contiguous, balanced shard r of n items over w workers: [n*r/w, n*(r+1)/w)  (mirrored for the CPU tests by tests/gloo_mirror.py: shard_bounds)
inline void shard_bounds(size_t n, int r, int w, size_t& lo, size_t& hi) {
    lo = n * (size_t)r / (size_t)w;
    hi = n * (size_t)(r + 1) / (size_t)w;
}

}  // namespace cb
