// windows64.cuh -- row windows of a CrsMatrix with 64-bit offsets, the layer under spmv64.cu and spgemm64.cu.
//
// Both paths run the 32-bit entry points per window of consecutive rows.  The cut is made once, on the device, by one thread
// doing one binary search per window (at most kMaxWindows of them); per window the layer keeps a 32-bit row map relative to
// the window's base, the first offset rounded down to a multiple of `align` entries.  A caller that streams the window's
// arrays by bulk copies asks for align = 4 (16-byte aligned `values + base`); one that reads them element by element asks for
// align = 1.  A second bound on prefixes P (SpGEMM: products per row) cuts a window where either bound is reached.
#pragma once
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace b200sp {

constexpr int kMaxWindows = 4096;
constexpr int64_t kDefaultWindow = (int64_t)INT32_MAX - 65536;  // entries per window, room for the kernels' round-ups

// cut failures, returned by cut_windows beside the B200SP_* codes
constexpr int kWindowRowOverLimit = -1;  // one row alone exceeds the limit
constexpr int kWindowsOverCap = -2;      // more than kMaxWindows windows

struct RowWindow {
  int r0 = 0, r1 = 0;   // rows [r0, r1)
  int64_t base = 0;     // row_ptr[r0] rounded down to a multiple of align: the entry the window's pointers are shifted by
  int64_t end = 0;      // row_ptr[r1]
  int64_t rel_off = 0;  // offset of the window's relative row map (r1 - r0 + 1 values) in RowWindows::rel, multiple of align
};

struct RowWindows {
  std::vector<RowWindow> win;
  DevArray<int> rel;     // relative row maps of all windows
  int64_t rel_size = 0;  // ints in rel
  void release(cudaStream_t st) {
    rel.release(st);
    rel_size = 0;
    win.clear();
  }
};

// range of the set_window entries
inline int check_window_limit(const char* entry, int64_t max_entries) {
  B200SP_REQUIRE(max_entries >= 8 && max_entries <= kDefaultWindow, "%s: %lld not in [8, %lld]", entry, (long long)max_entries,
                 (long long)kDefaultWindow);
  return B200SP_OK;
}

namespace {

// window k starts at row R_k with base_k = rp[R_k] & ~(align - 1) and ends at the largest R' with rp[R'] <= base_k + limit and,
// when P is given, P[R'] <= P[R_k] + limit.  out[4k .. 4k+3] = (R_k, R_{k+1}, base_k, rp[R_{k+1}]); status[0] = windows, or
// kWindowRowOverLimit (status[1] = the row) or kWindowsOverCap.
__global__ void win64_cut_kernel(int64_t m, const int64_t* __restrict__ rp, const int64_t* __restrict__ P, int64_t limit,
                                 int64_t align, int64_t* __restrict__ out, int64_t* __restrict__ status) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  int k = 0;
  int64_t R = 0;
  while (R < m) {
    const int64_t base = rp[R] & ~(align - 1);
    const int64_t top = base + limit, ptop = P ? P[R] + limit : 0;
    // largest R2 in (R, m] within both bounds; rp[R] - base < align <= limit, so lo = R always is
    int64_t lo = R, hi = m;
    while (lo < hi) {
      const int64_t mid = lo + ((hi - lo + 1) >> 1);
      if (rp[mid] <= top && (!P || P[mid] <= ptop)) lo = mid;
      else hi = mid - 1;
    }
    if (lo == R) {
      status[0] = kWindowRowOverLimit;
      status[1] = R;
      return;
    }
    if (k == kMaxWindows) {
      status[0] = kWindowsOverCap;
      return;
    }
    out[4 * k] = R;
    out[4 * k + 1] = lo;
    out[4 * k + 2] = base;
    out[4 * k + 3] = rp[lo];
    ++k;
    R = lo;
  }
  status[0] = k;
}

__global__ void __launch_bounds__(256) win64_relative_kernel(int64_t r0, int64_t count, int64_t base, const int64_t* __restrict__ rp,
                                                             int* __restrict__ rel) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
    rel[i] = (int)(rp[r0 + i] - base);
}

__global__ void __launch_bounds__(256) win64_widen_kernel(int64_t r0, int64_t count, int64_t base, const int* __restrict__ rel,
                                                          int64_t* __restrict__ rp) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
    rp[r0 + i] = base + rel[i];
}

// out = (int)in; *bad = 1 when a value does not fit 31 bits (bad may be null: values known to fit)
__global__ void __launch_bounds__(256) win64_narrow_kernel(int64_t n, const int64_t* __restrict__ in, int* __restrict__ out,
                                                           int* __restrict__ bad) {
  bool any = false;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t c = in[i];
    any |= (c < 0 || c > (int64_t)INT32_MAX);
    out[i] = (int)c;
  }
  if (any && bad) *bad = 1;
}

// Cuts rows [0, m) of rp (m + 1 offsets on the device; P, when given, m + 1 prefixes) and writes the windows' relative row
// maps into one array allocated here.  Returns B200SP_OK, kWindowRowOverLimit (*bad_row = the row), kWindowsOverCap or a
// CUDA error (message set); on failure *out is left empty and nothing stays allocated.  Two read-backs: count, records.
int cut_windows(cudaStream_t st, int64_t m, const int64_t* rp, const int64_t* P, int64_t limit, int align, RowWindows* out,
                int64_t* bad_row) {
  out->release(st);
  int64_t* d_rec;
  int64_t* d_status;
  int64_t status[2] = {0, 0};
  std::vector<int64_t> rec;
  {
    DevTmp tmp(st);
    B200SP_CUDA_TRY(tmp.alloc(&d_rec, (size_t)4 * kMaxWindows));
    B200SP_CUDA_TRY(tmp.alloc(&d_status, 2));
    win64_cut_kernel<<<1, 32, 0, st>>>(m, rp, P, limit, align, d_rec, d_status);
    B200SP_LAUNCH_CHECK();
    B200SP_CUDA_TRY(cudaMemcpyAsync(status, d_status, sizeof(status), cudaMemcpyDeviceToHost, st));
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
    if (status[0] == kWindowRowOverLimit) *bad_row = status[1];
    if (status[0] < 0) return (int)status[0];
    rec.resize((size_t)(4 * status[0]));
    if (status[0] > 0) {
      B200SP_CUDA_TRY(cudaMemcpyAsync(rec.data(), d_rec, sizeof(int64_t) * rec.size(), cudaMemcpyDeviceToHost, st));
      B200SP_CUDA_TRY(cudaStreamSynchronize(st));
    }
  }
  std::vector<RowWindow> win((size_t)status[0]);
  int64_t total = 0;
  for (size_t k = 0; k < win.size(); ++k) {
    RowWindow& w = win[k];
    w.r0 = (int)rec[4 * k];
    w.r1 = (int)rec[4 * k + 1];
    w.base = rec[4 * k + 2];
    w.end = rec[4 * k + 3];
    w.rel_off = total;
    total += ((int64_t)(w.r1 - w.r0) + 1 + align - 1) & ~(int64_t)(align - 1);
  }
  DevArray<int> rel;
  B200SP_CUDA_TRY(rel.alloc((size_t)std::max<int64_t>(total, 1), st));
  const int rc = [&]() -> int {
    for (const RowWindow& w : win) {
      const int64_t count = (int64_t)(w.r1 - w.r0) + 1;
      win64_relative_kernel<<<grid_for(count), 256, 0, st>>>(w.r0, count, w.base, rp, rel + w.rel_off);
      B200SP_LAUNCH_CHECK();
    }
    return B200SP_OK;
  }();
  if (rc) {
    rel.release(st);
    return rc;
  }
  out->win = std::move(win);
  out->rel = std::move(rel);
  out->rel_size = total;
  return B200SP_OK;
}

}  // namespace
}  // namespace b200sp
