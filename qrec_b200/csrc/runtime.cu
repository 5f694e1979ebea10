// Host-facing runtime: the call trainModel makes when the sampled triples live in HOST memory
// (the reference builds them as Python lists, base/deepRecommender.py:44-52, and hands them to
// sess.run(feed_dict) once per minibatch, model/ranking/LightGCN.py:38).  Here one call takes a
// whole epoch's index arrays, cuts them into chunks and runs a copy/compute pipeline:
//
//   copy stream   : H2D chunk c+1 (u,i,j) into ring slot (c+1)%R     | waits slot_free
//   compute stream: bpr_sgd_batch_kernel on ring slot c%R            | waits slot_ready
//
// so PCIe transfers hide behind the kernel (or vice versa, whichever is slower).
#include <vector>

#include "common.h"

struct qrec_ctx {
  int device = 0;
  long long chunk = 0;
  static constexpr int R = 3;
  int32_t* slot[R] = {nullptr, nullptr, nullptr};  // each 3*chunk ints: u | i | j
  int64_t* rp_slot[R] = {nullptr, nullptr, nullptr};  // each chunk+1 offsets (user-major epochs)
  cudaEvent_t ready[R], freed[R];
  cudaStream_t copy = nullptr, compute = nullptr;
  double* dev_loss = nullptr;
  double* pinned_loss = nullptr;
  const uint32_t* rated_sig = nullptr;   // optional [n_users, 16] rated-set signatures (qrec_rated_signature_build)
};

extern "C" {

int qrec_ctx_create(int device, int64_t chunk_triples, qrec_ctx** out) {
  QREC_REQUIRE(out != nullptr, "qrec_ctx_create: null out");
  QREC_REQUIRE(chunk_triples >= 0 && chunk_triples <= (1LL << 30), "qrec_ctx_create: bad chunk size");
  if (chunk_triples == 0) chunk_triples = 1 << 22;
  QREC_CUDA(cudaSetDevice(device));
  qrec_ctx* c = new (std::nothrow) qrec_ctx();
  if (!c) { qrec::set_error("qrec_ctx_create: out of host memory"); return QREC_ERR_NOMEM; }
  c->device = device;
  c->chunk = chunk_triples;
  QREC_CUDA(cudaStreamCreateWithFlags(&c->copy, cudaStreamNonBlocking));
  QREC_CUDA(cudaStreamCreateWithFlags(&c->compute, cudaStreamNonBlocking));
  for (int r = 0; r < qrec_ctx::R; ++r) {
    QREC_CUDA(cudaMalloc(&c->slot[r], sizeof(int32_t) * 3 * (size_t)chunk_triples));
    QREC_CUDA(cudaMalloc(&c->rp_slot[r], sizeof(int64_t) * ((size_t)chunk_triples + 1)));
    QREC_CUDA(cudaEventCreateWithFlags(&c->ready[r], cudaEventDisableTiming));
    QREC_CUDA(cudaEventCreateWithFlags(&c->freed[r], cudaEventDisableTiming));
  }
  QREC_CUDA(cudaMalloc(&c->dev_loss, sizeof(double)));
  QREC_CUDA(cudaMallocHost(&c->pinned_loss, sizeof(double)));
  *out = c;
  return QREC_OK;
}

int qrec_ctx_destroy(qrec_ctx* c) {
  if (!c) return QREC_OK;
  cudaSetDevice(c->device);
  if (c->copy) cudaStreamSynchronize(c->copy);
  if (c->compute) cudaStreamSynchronize(c->compute);
  for (int r = 0; r < qrec_ctx::R; ++r) {
    if (c->slot[r]) cudaFree(c->slot[r]);
    if (c->rp_slot[r]) cudaFree(c->rp_slot[r]);
    cudaEventDestroy(c->ready[r]);
    cudaEventDestroy(c->freed[r]);
  }
  if (c->dev_loss) cudaFree(c->dev_loss);
  if (c->pinned_loss) cudaFreeHost(c->pinned_loss);
  if (c->copy) cudaStreamDestroy(c->copy);
  if (c->compute) cudaStreamDestroy(c->compute);
  delete c;
  return QREC_OK;
}

int qrec_bpr_epoch_host(qrec_ctx* c, float* P, float* Q, int32_t d, int64_t n,
                        const int32_t* hu, const int32_t* hi, const int32_t* hj, float lr,
                        float reg_u, float reg_i, double* host_loss) {
  QREC_REQUIRE(c && P && Q && host_loss, "qrec_bpr_epoch_host: null pointer");
  QREC_REQUIRE(n >= 0 && (n == 0 || (hu && hi && hj)), "qrec_bpr_epoch_host: bad index arrays");
  QREC_CUDA(cudaSetDevice(c->device));
  QREC_CUDA(cudaMemsetAsync(c->dev_loss, 0, sizeof(double), c->compute));
  const long long chunk = c->chunk;
  long long done = 0;
  for (int it = 0; done < n; ++it, done += chunk) {
    const int r = it % qrec_ctx::R;
    const long long m = (n - done) < chunk ? (n - done) : chunk;
    int32_t* du = c->slot[r];
    int32_t* di = du + chunk;
    int32_t* dj = di + chunk;
    if (it >= qrec_ctx::R) QREC_CUDA(cudaStreamWaitEvent(c->copy, c->freed[r], 0));
    QREC_CUDA(cudaMemcpyAsync(du, hu + done, sizeof(int32_t) * (size_t)m, cudaMemcpyHostToDevice, c->copy));
    QREC_CUDA(cudaMemcpyAsync(di, hi + done, sizeof(int32_t) * (size_t)m, cudaMemcpyHostToDevice, c->copy));
    QREC_CUDA(cudaMemcpyAsync(dj, hj + done, sizeof(int32_t) * (size_t)m, cudaMemcpyHostToDevice, c->copy));
    QREC_CUDA(cudaEventRecord(c->ready[r], c->copy));
    QREC_CUDA(cudaStreamWaitEvent(c->compute, c->ready[r], 0));
    const int rc = qrec::launch_bpr_batch(P, Q, d, m, du, di, dj, lr, reg_u, reg_i, c->dev_loss, c->compute);
    if (rc != QREC_OK) return rc;
    QREC_CUDA(cudaEventRecord(c->freed[r], c->compute));
  }
  QREC_CUDA(cudaMemcpyAsync(c->pinned_loss, c->dev_loss, sizeof(double), cudaMemcpyDeviceToHost, c->compute));
  QREC_CUDA(cudaStreamSynchronize(c->compute));
  *host_loss = *c->pinned_loss;
  return QREC_OK;
}

// User-major epoch from HOST positives: host_rowptr (int64[n_users+1]) and host_i (int32[n]) are cut
// into chunks of whole users (<= chunk triples and <= chunk users each); chunk c+1 is copied on the copy
// stream while the fused sampling+SGD kernel runs chunk c.  The rejection CSR stays resident on the
// device; negatives are drawn in the kernel (Philox counter = global triple index, so the result does
// not depend on the chunking).
int qrec_ctx_set_rated_signature(qrec_ctx* c, const uint32_t* dev_sig) {
  QREC_REQUIRE(c != nullptr, "qrec_ctx_set_rated_signature: null ctx");
  c->rated_sig = dev_sig;
  return QREC_OK;
}

int qrec_bpr_epoch_usermajor_host(qrec_ctx* c, float* P, float* Q, int32_t d, int32_t n_users,
                                  const int64_t* host_rowptr, const int32_t* host_i,
                                  const int64_t* dev_rated_rowptr, const int32_t* dev_rated_cols,
                                  int32_t num_items, uint64_t seed, uint32_t epoch, float lr, float reg_u,
                                  float reg_i, double* host_loss) {
  QREC_REQUIRE(c && P && Q && host_loss, "qrec_bpr_epoch_usermajor_host: null pointer");
  QREC_REQUIRE(n_users >= 0 && (n_users == 0 || (host_rowptr && dev_rated_rowptr && dev_rated_cols)),
               "qrec_bpr_epoch_usermajor_host: bad arguments");
  QREC_CUDA(cudaSetDevice(c->device));
  QREC_CUDA(cudaMemsetAsync(c->dev_loss, 0, sizeof(double), c->compute));
  const long long chunk = c->chunk;
  int32_t ua = 0;
  for (int it = 0; ua < n_users; ++it) {
    // largest ub with rowptr[ub] - rowptr[ua] <= chunk and ub - ua <= chunk (at least one user)
    int32_t lo = ua + 1, hi = n_users;
    if ((long long)hi - ua > chunk) hi = (int32_t)(ua + chunk);
    while (lo < hi) {
      const int32_t mid = lo + (hi - lo + 1) / 2;
      if (host_rowptr[mid] - host_rowptr[ua] <= chunk) lo = mid; else hi = mid - 1;
    }
    const int32_t ub = lo;
    const long long t0 = host_rowptr[ua], m = host_rowptr[ub] - t0;
    QREC_REQUIRE(m <= chunk, "qrec_bpr_epoch_usermajor_host: user %d has %lld positives, more than the ctx chunk (%lld)",
                 ua, (long long)m, chunk);
    const int r = it % qrec_ctx::R;
    if (it >= qrec_ctx::R) QREC_CUDA(cudaStreamWaitEvent(c->copy, c->freed[r], 0));
    QREC_CUDA(cudaMemcpyAsync(c->rp_slot[r], host_rowptr + ua, sizeof(int64_t) * (size_t)(ub - ua + 1),
                              cudaMemcpyHostToDevice, c->copy));
    if (m > 0) QREC_CUDA(cudaMemcpyAsync(c->slot[r], host_i + t0, sizeof(int32_t) * (size_t)m, cudaMemcpyHostToDevice, c->copy));
    QREC_CUDA(cudaEventRecord(c->ready[r], c->copy));
    QREC_CUDA(cudaStreamWaitEvent(c->compute, c->ready[r], 0));
    if (m > 0) {
      const int rc = qrec::launch_usermajor(P + (size_t)ua * d, Q, d, ub - ua, m, c->rp_slot[r], c->slot[r], nullptr, lr,
                                            reg_u, reg_i, c->dev_loss, true, dev_rated_rowptr + ua, dev_rated_cols,
                                            num_items, seed, epoch, nullptr, t0, c->compute,
                                            c->rated_sig ? c->rated_sig + (size_t)ua * 16 : nullptr);
      if (rc != QREC_OK) return rc;
    }
    QREC_CUDA(cudaEventRecord(c->freed[r], c->compute));
    ua = ub;
  }
  QREC_CUDA(cudaMemcpyAsync(c->pinned_loss, c->dev_loss, sizeof(double), cudaMemcpyDeviceToHost, c->compute));
  QREC_CUDA(cudaStreamSynchronize(c->compute));
  *host_loss = *c->pinned_loss;
  return QREC_OK;
}

}  // extern "C"
