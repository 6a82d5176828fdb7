// Host-buffer entry points: H2D staging -> kernels -> D2H result, one blocking call.
#include <cuda_runtime.h>

#include "../../include/sbi_b200.h"
#include "device.cuh"

#define CK(x)                            \
  do {                                   \
    cudaError_t e_ = (x);                \
    if (e_ != cudaSuccess) return (int)e_; \
  } while (0)

// forward+backward of the staged batch: tensor-core kernels when the workspace carries their operand
// descriptors, else the SIMT kernel, which spills its activations to ws->d_save when the workspace has one.
// Returns the number of partial-gradient slabs written in *n_part.
static int vjp_staged(const sbi_nsf_model* m, const sbi_train_ws* ws, int64_t B, float g_const, int* n_part,
                      void* stream) {
  sbi_rows rows;
  rows.d_input = ws->d_input;
  rows.d_cond = ws->d_cond;
  rows.d_index = nullptr;
  rows.R = B;
  rows.cond_shared = 0;
  if (ws->tc_fwd != nullptr && ws->tc_bwd != nullptr && ws->tc_pack != nullptr && ws->d_save != nullptr) {
    int rc = sbi_b200_nsf_tc_pack(m, ws->tc_pack, stream);
    if (rc) return rc;
    *n_part = sbi_b200_nsf_vjp_tc_parts(B);
    return sbi_b200_nsf_vjp_tc(m, ws->tc_fwd, ws->tc_bwd, &rows, nullptr, g_const, nullptr, ws->d_gpart,
                               ws->d_loss_acc, ws->d_save, ws->save_bytes, stream);
  }
  *n_part = sbi_b200_nsf_vjp_parts(B);
  return sbi_b200_nsf_vjp(m, &rows, nullptr, g_const, nullptr, ws->d_gpart, nullptr, nullptr, ws->d_loss_acc,
                          ws->d_save, ws->save_bytes, stream);
}

// partial-gradient reduction (+ per-block sum of squares when the workspace has room) -> clip + Adam
static int reduce_and_step(const sbi_nsf_model* m, const sbi_train_ws* ws, int n_part, float lr, float beta1,
                           float beta2, float eps, float max_norm, void* stream) {
  if (ws->d_sumsq != nullptr) {
    int rc = sbi_b200_reduce_partials_norm(ws->d_gpart, n_part, m->n_params, ws->d_grad, ws->d_mask,
                                           ws->d_sumsq, stream);
    if (rc) return rc;
    return sbi_b200_adam_clip_step_norm(const_cast<float*>(m->d_params), ws->d_grad, ws->d_state, ws->d_step,
                                        ws->d_mask, m->n_params, lr, beta1, beta2, eps, max_norm, 1.0f,
                                        ws->d_sumsq, sbi_b200_sumsq_blocks(m->n_params), stream);
  }
  int rc = sbi_b200_reduce_partials(ws->d_gpart, n_part, m->n_params, ws->d_grad, stream);
  if (rc) return rc;
  return sbi_b200_adam_clip_step(const_cast<float*>(m->d_params), ws->d_grad, ws->d_state, ws->d_step,
                                 ws->d_mask, m->n_params, lr, beta1, beta2, eps, max_norm, 1.0f, stream);
}

extern "C" int sbi_b200_nsf_train_step_host(const sbi_nsf_model* m, const sbi_train_ws* ws,
                                            const float* h_input, const float* h_cond, int64_t B,
                                            float lr, float beta1, float beta2, float eps,
                                            float max_norm, float* h_loss_out, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  if (!m || !ws || !h_input || !h_cond || !h_loss_out || B < 1 || B > ws->cap_rows)
    return SBI_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaMemcpyAsync(ws->d_input, h_input, sizeof(float) * B * m->D, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ws->d_cond, h_cond, sizeof(float) * B * m->C, cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(ws->d_loss_acc, 0, 2 * sizeof(float), s));
  int n_part = 0;
  int rc = vjp_staged(m, ws, B, -1.0f / (float)B, &n_part, stream);
  if (rc) return rc;
  rc = reduce_and_step(m, ws, n_part, lr, beta1, beta2, eps, max_norm, stream);
  if (rc) return rc;
  CK(cudaMemcpyAsync(h_loss_out, ws->d_loss_acc, 2 * sizeof(float), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int sbi_b200_nsf_logprob_host(const sbi_nsf_model* m, const sbi_train_ws* ws,
                                         const float* h_input, const float* h_cond, int64_t R,
                                         int cond_shared, float* h_logp, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  if (!m || !ws || !h_input || !h_cond || !h_logp || R < 1 || R > ws->cap_rows) return SBI_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaMemcpyAsync(ws->d_input, h_input, sizeof(float) * R * m->D, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ws->d_cond, h_cond, sizeof(float) * (cond_shared ? 1 : R) * m->C,
                     cudaMemcpyHostToDevice, s));
  sbi_rows rows;
  rows.d_input = ws->d_input;
  rows.d_cond = ws->d_cond;
  rows.d_index = nullptr;
  rows.R = R;
  rows.cond_shared = cond_shared ? 1 : 0;
  int rc = sbi_b200_nsf_logprob(m, &rows, ws->d_logp, nullptr, stream);
  if (rc) return rc;
  CK(cudaMemcpyAsync(h_logp, ws->d_logp, sizeof(float) * R, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return 0;
}

// Host rows through the tensor-core kernel, chunked over two internal streams so that the H2D
// copy of chunk i+1 and the D2H copy of chunk i-1 overlap the kernel of chunk i.  The operands are
// re-packed first (tc->d_tcw).  Ordered after prior work on `stream`; returns when h_logp is
// complete.
extern "C" int sbi_b200_nsf_logprob_host_tc(const sbi_nsf_model* m, const sbi_nsf_tc* tc,
                                            const sbi_train_ws* ws, const float* h_input,
                                            const float* h_cond, int64_t R, int cond_shared,
                                            float* h_logp, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  if (!m || !tc || !ws || !h_input || !h_cond || !h_logp || R < 1 || R > ws->cap_rows) return SBI_EINVAL;
  if (!sbi_b200_nsf_tc_supported(m, tc)) return SBI_ESMEM;
  static cudaStream_t ss[2] = {nullptr, nullptr};
  static cudaEvent_t ev_in = nullptr, ev_out[2] = {nullptr, nullptr};
  if (!ss[0]) {
    for (int i = 0; i < 2; ++i) {
      CK(cudaStreamCreateWithFlags(&ss[i], cudaStreamNonBlocking));
      CK(cudaEventCreateWithFlags(&ev_out[i], cudaEventDisableTiming));
    }
    CK(cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming));
  }
  cudaStream_t s = (cudaStream_t)stream;
  int rc = sbi_b200_nsf_tc_pack(m, tc, stream);
  if (rc) return rc;
  if (cond_shared)
    CK(cudaMemcpyAsync(ws->d_cond, h_cond, sizeof(float) * m->C, cudaMemcpyHostToDevice, s));
  CK(cudaEventRecord(ev_in, s));
  CK(cudaStreamWaitEvent(ss[0], ev_in, 0));
  CK(cudaStreamWaitEvent(ss[1], ev_in, 0));
  const int64_t chunk = 1 << 17;   // 128 Ki rows: ~0.3 ms of kernel, 5 MB of input
  int k = 0;
  for (int64_t r0 = 0; r0 < R; r0 += chunk, k ^= 1) {
    const int64_t n = (R - r0 < chunk) ? R - r0 : chunk;
    CK(cudaMemcpyAsync(ws->d_input + r0 * m->D, h_input + r0 * m->D, sizeof(float) * n * m->D,
                       cudaMemcpyHostToDevice, ss[k]));
    if (!cond_shared)
      CK(cudaMemcpyAsync(ws->d_cond + r0 * m->C, h_cond + r0 * m->C, sizeof(float) * n * m->C,
                         cudaMemcpyHostToDevice, ss[k]));
    sbi_rows rows;
    rows.d_input = ws->d_input + r0 * m->D;
    rows.d_cond = cond_shared ? ws->d_cond : ws->d_cond + r0 * m->C;
    rows.d_index = nullptr;
    rows.R = n;
    rows.cond_shared = cond_shared ? 1 : 0;
    rc = sbi_b200_nsf_logprob_tc(m, tc, &rows, ws->d_logp + r0, nullptr, (void*)ss[k]);
    if (rc) return rc;
    CK(cudaMemcpyAsync(h_logp + r0, ws->d_logp + r0, sizeof(float) * n, cudaMemcpyDeviceToHost, ss[k]));
  }
  for (int i = 0; i < 2; ++i) {
    CK(cudaEventRecord(ev_out[i], ss[i]));
    CK(cudaStreamWaitEvent(s, ev_out[i], 0));
  }
  CK(cudaStreamSynchronize(s));
  return 0;
}

// ---- pipelined host steps ------------------------------------------------------------------------
struct SbiPipe {
  cudaEvent_t done[2];
  float* h_loss[2];   // pinned
  int64_t n;          // steps enqueued
};

extern "C" void* sbi_b200_pipe_create(void) {
  SbiPipe* p = new SbiPipe();
  p->n = 0;
  for (int i = 0; i < 2; ++i) {
    if (cudaEventCreateWithFlags(&p->done[i], cudaEventDisableTiming) != cudaSuccess) return nullptr;
    if (cudaMallocHost(&p->h_loss[i], 2 * sizeof(float)) != cudaSuccess) return nullptr;
  }
  return p;
}

extern "C" void sbi_b200_pipe_destroy(void* pipe) {
  sbi::DeviceGuard dev_guard_(pipe);
  SbiPipe* p = static_cast<SbiPipe*>(pipe);
  if (!p) return;
  for (int i = 0; i < 2; ++i) {
    cudaEventDestroy(p->done[i]);
    cudaFreeHost(p->h_loss[i]);
  }
  delete p;
}

static int pipe_wait_prev(SbiPipe* p, float* h_out) {
  if (p->n == 0) {
    if (h_out) h_out[0] = h_out[1] = nanf("");
    return 0;
  }
  const int s = (int)((p->n - 1) & 1);
  CK(cudaEventSynchronize(p->done[s]));
  if (h_out) { h_out[0] = p->h_loss[s][0]; h_out[1] = p->h_loss[s][1]; }
  return 0;
}

extern "C" int sbi_b200_nsf_train_step_host_async(const sbi_nsf_model* m, const sbi_train_ws* ws, void* pipe,
                                                  const float* h_input, const float* h_cond, int64_t B,
                                                  float lr, float beta1, float beta2, float eps,
                                                  float max_norm, float* h_loss_prev, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  SbiPipe* p = static_cast<SbiPipe*>(pipe);
  if (!m || !ws || !p || !h_input || !h_cond || B < 1 || B > ws->cap_rows) return SBI_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const int slot = (int)(p->n & 1);
  CK(cudaMemcpyAsync(ws->d_input, h_input, sizeof(float) * B * m->D, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ws->d_cond, h_cond, sizeof(float) * B * m->C, cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(ws->d_loss_acc, 0, 2 * sizeof(float), s));
  int n_part = 0;
  int rc = vjp_staged(m, ws, B, -1.0f / (float)B, &n_part, stream);
  if (rc) return rc;
  rc = reduce_and_step(m, ws, n_part, lr, beta1, beta2, eps, max_norm, stream);
  if (rc) return rc;
  CK(cudaMemcpyAsync(p->h_loss[slot], ws->d_loss_acc, 2 * sizeof(float), cudaMemcpyDeviceToHost, s));
  CK(cudaEventRecord(p->done[slot], s));
  rc = pipe_wait_prev(p, h_loss_prev);   // step i-1 (the other slot) -- this step keeps running
  p->n += 1;
  return rc;
}

// Data-parallel variant of the pipelined host step (one process per GPU): between the reduction
// of the per-CTA partial gradients and clip+Adam the flat gradients of all ranks are summed over
// NVLink peer memory (sbi_b200_peer_sum, csrc/peer.cu; it also emits the sum(g^2) partials).  The
// upstream gradient is -1/(B * world): rows of all ranks form one global batch.
extern "C" int sbi_b200_nsf_train_step_host_async_dp(const sbi_nsf_model* m, const sbi_train_ws* ws, void* pipe,
                                                     const sbi_peer_ctx* peer, const float* h_input,
                                                     const float* h_cond, int64_t B, float lr, float beta1,
                                                     float beta2, float eps, float max_norm,
                                                     float* h_loss_prev, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  SbiPipe* p = static_cast<SbiPipe*>(pipe);
  if (!m || !ws || !p || !peer || !peer->h_peer_ptrs || !peer->d_grad_local || !ws->d_sumsq || !h_input ||
      !h_cond || B < 1 || B > ws->cap_rows || peer->world < 1)
    return SBI_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const int slot = (int)(p->n & 1);
  CK(cudaMemcpyAsync(ws->d_input, h_input, sizeof(float) * B * m->D, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ws->d_cond, h_cond, sizeof(float) * B * m->C, cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(ws->d_loss_acc, 0, 2 * sizeof(float), s));
  int n_part = 0;
  int rc = vjp_staged(m, ws, B, -1.0f / ((float)B * (float)peer->world), &n_part, stream);
  if (rc) return rc;
  rc = sbi_b200_reduce_partials(ws->d_gpart, n_part, m->n_params, peer->d_grad_local, stream);
  if (rc) return rc;
  rc = sbi_b200_peer_sum(peer->d_grad_local, peer->h_peer_ptrs, peer->world, peer->rank, m->n_params,
                         ws->d_grad, ws->d_mask, ws->d_sumsq, nullptr, stream);
  if (rc) return rc;
  rc = sbi_b200_adam_clip_step_norm(const_cast<float*>(m->d_params), ws->d_grad, ws->d_state, ws->d_step,
                                    ws->d_mask, m->n_params, lr, beta1, beta2, eps, max_norm, 1.0f,
                                    ws->d_sumsq, sbi_b200_peer_blocks(m->n_params), stream);
  if (rc) return rc;
  CK(cudaMemcpyAsync(p->h_loss[slot], ws->d_loss_acc, 2 * sizeof(float), cudaMemcpyDeviceToHost, s));
  CK(cudaEventRecord(p->done[slot], s));
  rc = pipe_wait_prev(p, h_loss_prev);
  p->n += 1;
  return rc;
}

extern "C" int sbi_b200_pipe_drain(void* pipe, float* h_loss_last) {
  sbi::DeviceGuard dev_guard_(pipe);
  SbiPipe* p = static_cast<SbiPipe*>(pipe);
  if (!p) return SBI_EINVAL;
  return pipe_wait_prev(p, h_loss_last);
}
