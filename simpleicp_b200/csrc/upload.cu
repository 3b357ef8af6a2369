// upload.cu — see upload.cuh.
#include "upload.cuh"

#include <cstring>

#include "common.cuh"

namespace sicp {

bool PageableUploader::is_pageable(const void* p) {
  if (!p) return false;
  cudaPointerAttributes at;
  const cudaError_t e = cudaPointerGetAttributes(&at, p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return at.type == cudaMemoryTypeUnregistered;
}

void PageableUploader::run_share(int t, const Job& job) {
  int use = 0;
  for (size_t j = (size_t)t; j < job.n_chunks; j += (size_t)job.n_threads, ++use) {
    const int b = use % kBuffers;
    const size_t off = j * job.chunk, len = (off + job.chunk <= job.bytes) ? job.chunk : job.bytes - off;
    // the buffer's previous DMA — of this transfer or of an earlier one — must have left it
    // (an event that was never recorded completes at once)
    cudaError_t e = cudaEventSynchronize(ev_[t][b]);
    if (e == cudaSuccess) {
      std::memcpy(stage_[t][b], job.src + off, len);
      e = cudaMemcpyAsync(job.dst + off, stage_[t][b], len, cudaMemcpyHostToDevice, ws_[t]);
    }
    if (e == cudaSuccess) e = cudaEventRecord(ev_[t][b], ws_[t]);
    if (e != cudaSuccess) {
      err_.store((int)e | 0x10000);
      return;
    }
  }
  const cudaError_t e = cudaEventRecord(done_[t], ws_[t]);
  if (e != cudaSuccess) err_.store((int)e | 0x10000);
}

void PageableUploader::worker(int t, uint64_t seen) {
  const bool bound = cudaSetDevice(device_) == cudaSuccess;
  for (;;) {
    Job job;
    {
      std::unique_lock<std::mutex> lk(m_);
      cv_work_.wait(lk, [&] { return quit_ || job_id_ != seen; });
      if (quit_) return;
      seen = job_id_;
      job = job_;
    }
    if (t < job.n_threads) {
      if (bound) run_share(t, job);
      else err_.store((int)cudaErrorInvalidDevice | 0x10000);
    }
    {
      std::lock_guard<std::mutex> lk(m_);
      if (--pending_ == 0) cv_done_.notify_all();
    }
  }
}

void PageableUploader::ensure(int device, int n_threads) {
  if (device_ != device && !pool_.empty())
    throw Error{SICP_ERR_STATE, "pageable uploader used on two devices"};
  device_ = device;
  while ((int)pool_.size() < n_threads) {
    const int t = (int)pool_.size();
    SICP_CUDA(cudaStreamCreateWithFlags(&ws_[t], cudaStreamNonBlocking));
    SICP_CUDA(cudaEventCreateWithFlags(&done_[t], cudaEventDisableTiming));
    for (int b = 0; b < kBuffers; ++b) {
      SICP_CUDA(cudaHostAlloc(&stage_[t][b], kStage, cudaHostAllocDefault));
      SICP_CUDA(cudaEventCreateWithFlags(&ev_[t][b], cudaEventDisableTiming));
    }
    uint64_t seen;
    {
      std::lock_guard<std::mutex> lk(m_);
      seen = job_id_;  // a new worker never picks up a job that was posted before it existed
    }
    pool_.emplace_back(&PageableUploader::worker, this, t, seen);
  }
}

void PageableUploader::start(int device, int n_threads, void* dst, const void* src, size_t bytes,
                             cudaEvent_t after) {
  abandon();  // a previous transfer that was never finished (error path): wait for it first
  if (bytes == 0) return;
  n_threads = n_threads < 1 ? 1 : (n_threads > kMaxThreads ? kMaxThreads : n_threads);
  const size_t ck = chunk < 65536 ? 65536 : (chunk > kStage ? kStage : chunk);
  const size_t n_chunks = (bytes + ck - 1) / ck;
  if ((size_t)n_threads > n_chunks) n_threads = (int)n_chunks;
  ensure(device, n_threads);
  err_.store(0);
  if (after)
    for (int t = 0; t < n_threads; ++t) SICP_CUDA(cudaStreamWaitEvent(ws_[t], after, 0));
  {
    std::lock_guard<std::mutex> lk(m_);
    job_.dst = static_cast<unsigned char*>(dst);
    job_.src = static_cast<const unsigned char*>(src);
    job_.bytes = bytes;
    job_.n_chunks = n_chunks;
    job_.chunk = ck;
    job_.n_threads = n_threads;
    pending_ = (int)pool_.size();
    ++job_id_;
    n_used_ = n_threads;
    in_flight_ = true;
  }
  cv_work_.notify_all();
}

void PageableUploader::abandon() noexcept {
  if (!in_flight_) return;
  std::unique_lock<std::mutex> lk(m_);
  cv_done_.wait(lk, [&] { return pending_ == 0; });
  in_flight_ = false;
}

void PageableUploader::cancel() noexcept {
  abandon();
  for (int t = 0; t < n_used_; ++t) cudaStreamSynchronize(ws_[t]);
}

void PageableUploader::finish(cudaStream_t target) {
  if (!in_flight_) return;
  abandon();
  const int e = err_.load();
  if (e != 0)
    throw Error{SICP_ERR_CUDA, std::string("pageable upload failed: ") +
                                   cudaGetErrorString((cudaError_t)(e & 0xffff))};
  for (int t = 0; t < n_used_; ++t) SICP_CUDA(cudaStreamWaitEvent(target, done_[t], 0));
}

PageableUploader::~PageableUploader() {
  abandon();
  {
    std::lock_guard<std::mutex> lk(m_);
    quit_ = true;
  }
  cv_work_.notify_all();
  for (auto& th : pool_)
    if (th.joinable()) th.join();
  if (!pool_.empty() && device_ >= 0) cudaSetDevice(device_);
  for (size_t t = 0; t < pool_.size(); ++t) {
    if (ws_[t]) cudaStreamSynchronize(ws_[t]);
    for (int b = 0; b < kBuffers; ++b) {
      if (ev_[t][b]) cudaEventDestroy(ev_[t][b]);
      if (stage_[t][b]) cudaFreeHost(stage_[t][b]);
    }
    if (done_[t]) cudaEventDestroy(done_[t]);
    if (ws_[t]) cudaStreamDestroy(ws_[t]);
  }
}

}  // namespace sicp
