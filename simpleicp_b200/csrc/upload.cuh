// upload.cuh — host->device transfer of a caller's cloud when it lives in PAGEABLE host memory.
//
// cudaMemcpyAsync from pageable memory is staged by the driver through its own bounce buffer on
// the CALLING thread: 13-16 GB/s on this pool's hosts, and the call does not return before the
// source has been read, so nothing the library queues afterwards overlaps it.  NumPy arrays are
// pageable, i.e. this is the path of simpleicp(X_fix, X_mov) and SimpleICP.run() for every caller
// who does not pin memory.  Here a few persistent worker threads copy 2 MB slices into pinned
// staging buffers and queue the DMA of each slice themselves (one stream per worker, two
// buffers per worker), and the calling thread is free to queue kernels meanwhile.  Measured on
// the C3 pair (tools/upload_probe.py, 24 MB per cloud): 1.05-1.15 ms per cloud with 2, 3 or 4
// workers against 1.3-1.7 ms for the driver's path (0.44 ms from pinned memory);
// simpleicp(X_fix, X_mov) on NumPy arrays 5.4-6.2 -> 4.4-4.8 ms, because the second cloud now
// also crosses PCIe while the normals are computed.  Pinned and device sources keep the single
// cudaMemcpyAsync.
#pragma once
#include <atomic>
#include <condition_variable>
#include <cstddef>
#include <cstdint>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include <cuda_runtime.h>

namespace sicp {

struct PageableUploader {
  static constexpr int kMaxThreads = 8;
  static constexpr int kBuffers = 2;
  static constexpr size_t kStage = 4u << 20;  // size of one pinned staging buffer
  size_t chunk = 2u << 20;                    // slice size (<= kStage); option "upload_chunk_kb"

  ~PageableUploader();
  // true if p is ordinary (unregistered) host memory
  static bool is_pageable(const void* p);
  // Start copying bytes from src (pageable host) to dst (device) on the worker streams, which
  // first wait for `after` (may be null).  Returns at once; src must stay valid until finish().
  void start(int device, int n_threads, void* dst, const void* src, size_t bytes, cudaEvent_t after);
  // Wait for the workers (host side: src has been read completely) and make `target` wait for
  // their transfers (device side).  Throws sicp::Error if a worker failed.  No-op when idle.
  void finish(cudaStream_t target);
  // Host-side wait only: never throws.
  void abandon() noexcept;
  // Error paths: abandon(), then wait until the DMA the workers queued has landed.  The failing
  // call may not have made any stream wait for it, and the next call may copy into the same
  // device buffer from another stream.  Never throws.
  void cancel() noexcept;
  bool active() const { return in_flight_; }

 private:
  struct Job {
    unsigned char* dst = nullptr;
    const unsigned char* src = nullptr;
    size_t bytes = 0, n_chunks = 0, chunk = 0;
    int n_threads = 0;
  };
  void ensure(int device, int n_threads);
  void worker(int t, uint64_t seen);
  void run_share(int t, const Job& job);

  int device_ = -1;
  cudaStream_t ws_[kMaxThreads] = {};
  void* stage_[kMaxThreads][kBuffers] = {};
  cudaEvent_t ev_[kMaxThreads][kBuffers] = {};
  cudaEvent_t done_[kMaxThreads] = {};
  std::vector<std::thread> pool_;
  std::mutex m_;
  std::condition_variable cv_work_, cv_done_;
  Job job_;
  uint64_t job_id_ = 0;
  int pending_ = 0;
  bool quit_ = false;
  bool in_flight_ = false;
  int n_used_ = 0;
  std::atomic<int> err_{0};
};

}  // namespace sicp
