// Host-buffer rollout shared by the three env families (the `*_rollout_host` entry points).
//
// The caller hands HOST pointers (pinned for full speed); the copies are part of the call.  The
// rollout is cut into chunks of lockstep steps: chunk c+1 is computed on one stream while the copy
// engines drain chunk c's trajectory rows on another, and the action upload rides in front on the
// compute stream (H2D and D2H use different copy engines).  With the full observation tensor
// returned, the call runs at the PCIe D2H rate (the kernel is ~1.5 % of it); with
// MADRL_HOST_OBS_LAST (policy on the device: only the last step's observations are needed on the
// host to continue) it runs at the kernel's rate.
#pragma once
#include "common.cuh"

namespace madrl {

struct HostPipe {
  void* stage = nullptr;
  size_t stage_bytes = 0;
  cudaStream_t compute = nullptr, copy = nullptr;
  cudaEvent_t done[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};

  // Blocking (default-flag) streams: ordered after earlier work on the legacy default stream (e.g. a
  // reset launched there), unordered with each other.
  int ensure(size_t bytes) {
    if (!compute) {
      MADRL_CUDA_CHECK(cudaStreamCreate(&compute));
      MADRL_CUDA_CHECK(cudaStreamCreate(&copy));
      for (int i = 0; i < 8; ++i) MADRL_CUDA_CHECK(cudaEventCreateWithFlags(&done[i], cudaEventDisableTiming));
    }
    if (stage_bytes >= bytes) return MADRL_OK;
    if (stage) cudaFree(stage);
    stage = nullptr;
    stage_bytes = 0;
    cudaError_t e = cudaMalloc(&stage, bytes);
    if (e != cudaSuccess) { set_error("cudaMalloc(stage %zu): %s", bytes, cudaGetErrorString(e)); return MADRL_ENOMEM; }
    stage_bytes = bytes;
    return MADRL_OK;
  }
  void destroy() {
    if (stage) cudaFree(stage);
    if (compute) cudaStreamDestroy(compute);
    if (copy) cudaStreamDestroy(copy);
    for (int i = 0; i < 8; ++i) if (done[i]) cudaEventDestroy(done[i]);
    stage = nullptr; compute = copy = nullptr;
  }
};

// Bytes of ONE lockstep step of each trajectory tensor (all tensors are time-major, so a chunk of
// steps is one contiguous slice of each).
struct StepBytes { size_t act, obs, rew, done, info; };

// launch(Tc, act_dev, obs_dev, rew_dev, done_dev, info_dev, stream) -> rc runs the next Tc lockstep steps.
template <class Launch>
int host_rollout(HostPipe& hp, int T, const StepBytes& sb, const void* act_h, void* obs_h, void* rew_h, void* done_h,
                 void* info_h, int obs_last_only, Launch launch) {
  const size_t TT = (size_t)T;
  const size_t o_obs = align_up(TT * sb.act, 256), o_rew = align_up(o_obs + TT * sb.obs, 256);
  const size_t o_done = align_up(o_rew + TT * sb.rew, 256), o_info = align_up(o_done + TT * sb.done, 256);
  int rc = hp.ensure(o_info + TT * sb.info);
  if (rc) return rc;
  char* st = (char*)hp.stage;
  // chunks of >= 32 MB (madrl_set_host_chunk_bytes) of device->host traffic -- below that a copy is
  // latency-dominated -- and at most 8
  const size_t out_step = (obs_last_only ? 0 : sb.obs) + sb.rew + sb.done + sb.info;
  size_t n_chunks = (TT * out_step) / g_host_chunk_bytes.load();
  if (n_chunks < 1) n_chunks = 1;
  if (n_chunks > 8) n_chunks = 8;
  if (n_chunks > TT) n_chunks = TT;
  // done / info rows are sliced at chunk boundaries: keep the 8-byte alignment of the info rows
  size_t Tc = (TT + n_chunks - 1) / n_chunks;
  while ((Tc * sb.info) % 8 != 0) ++Tc;
  MADRL_CUDA_CHECK(cudaMemcpyAsync(st, act_h, TT * sb.act, cudaMemcpyHostToDevice, hp.compute));
  int c = 0;
  for (size_t t0 = 0; t0 < TT; t0 += Tc, ++c) {
    const size_t n = (t0 + Tc <= TT) ? Tc : TT - t0;
    rc = launch((int)n, st + t0 * sb.act, st + o_obs + t0 * sb.obs, st + o_rew + t0 * sb.rew,
                st + o_done + t0 * sb.done, st + o_info + t0 * sb.info, hp.compute);
    if (rc) return rc;
    MADRL_CUDA_CHECK(cudaEventRecord(hp.done[c], hp.compute));
    MADRL_CUDA_CHECK(cudaStreamWaitEvent(hp.copy, hp.done[c], 0));
    if (!obs_last_only)
      MADRL_CUDA_CHECK(cudaMemcpyAsync((char*)obs_h + t0 * sb.obs, st + o_obs + t0 * sb.obs, n * sb.obs,
                                       cudaMemcpyDeviceToHost, hp.copy));
    else if (t0 + n == TT)
      MADRL_CUDA_CHECK(cudaMemcpyAsync(obs_h, st + o_obs + (TT - 1) * sb.obs, sb.obs, cudaMemcpyDeviceToHost, hp.copy));
    MADRL_CUDA_CHECK(cudaMemcpyAsync((char*)rew_h + t0 * sb.rew, st + o_rew + t0 * sb.rew, n * sb.rew,
                                     cudaMemcpyDeviceToHost, hp.copy));
    MADRL_CUDA_CHECK(cudaMemcpyAsync((char*)done_h + t0 * sb.done, st + o_done + t0 * sb.done, n * sb.done,
                                     cudaMemcpyDeviceToHost, hp.copy));
    MADRL_CUDA_CHECK(cudaMemcpyAsync((char*)info_h + t0 * sb.info, st + o_info + t0 * sb.info, n * sb.info,
                                     cudaMemcpyDeviceToHost, hp.copy));
  }
  MADRL_CUDA_CHECK(cudaStreamSynchronize(hp.copy));
  MADRL_CUDA_CHECK(cudaStreamSynchronize(hp.compute));
  return MADRL_OK;
}

}  // namespace madrl
