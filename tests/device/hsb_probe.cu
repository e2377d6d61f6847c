// hsb_probe.cu — the kernels' scalar device functions on their own, for the tests (not product code).
//
// Each entry point runs one production __device__ function elementwise over its arguments and returns the function's
// results: sinf_glibc / cosf_glibc / sincosf_glibc / expf_glibc (csrc/sincosf_glibc.h), normalize_angle,
// pose_difference_larger_than, solve3 and best_pack / best_unpack (csrc/match_kernel.cuh).  Nothing here computes a
// value itself: every output is what a call to the production function returned, so a test that compares these outputs
// with a host reference tests the device build of that function.  The library is compiled with the product library's
// nvcc flags (hector_slam_b200/build.py build_probe), so the code generation — -fmad=false above all — is the product's.
//
// C ABI, host buffers: each call copies its inputs to the device, launches, copies the outputs back and synchronises
// before it returns.  Returns 0, or the CUDA error code.  The unary sweeps take their arguments as a run of bit
// patterns (first, first + 1, ..., first + n - 1, wrapping at 2^32), generated on the device, so an exhaustive sweep
// moves only its outputs.  The product library never loads this one.
#include <cuda_runtime.h>
#include <stdint.h>

#include "match_kernel.cuh"
#include "sincosf_glibc.h"

namespace {

__device__ __forceinline__ float arg_of(uint32_t first, long long i) { return __uint_as_float(first + (uint32_t)i); }

__global__ void trig_kernel(uint32_t first, long long n, float* s, float* c, float* ss, float* sc) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float x = arg_of(first, i);
    s[i] = hsb::sinf_glibc(x);
    c[i] = hsb::cosf_glibc(x);
    float a, b;
    hsb::sincosf_glibc(x, &a, &b);
    ss[i] = a;
    sc[i] = b;
  }
}

__global__ void exp_kernel(uint32_t first, long long n, float* e) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    e[i] = hsb::expf_glibc(arg_of(first, i));
}

__global__ void norm_sweep_kernel(uint32_t first, long long n, float* na) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    na[i] = hsb::normalize_angle(arg_of(first, i));
}

__global__ void norm_kernel(const float* in, long long n, float* out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = hsb::normalize_angle(in[i]);
}

// h: n x 6 symmetric H as (h00, h11, h22, h01, h02, h12); d: n x 3 dTr; out: n x 3
__global__ void solve3_kernel(const float* h, const float* d, long long n, float* out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    hsb::Acc a;
    a.h00 = h[6 * i]; a.h11 = h[6 * i + 1]; a.h22 = h[6 * i + 2];
    a.h01 = h[6 * i + 3]; a.h02 = h[6 * i + 4]; a.h12 = h[6 * i + 5];
    a.d0 = d[3 * i]; a.d1 = d[3 * i + 1]; a.d2 = d[3 * i + 2];
    hsb::solve3(a, out[3 * i], out[3 * i + 1], out[3 * i + 2]);
  }
}

__global__ void gate_kernel(const float* p1, const float* p2, const float* dist, const float* ang, long long n, int* out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = hsb::pose_difference_larger_than(p1 + 3 * i, p2 + 3 * i, dist[i], ang[i]) ? 1 : 0;
}

// best_pack of (score, pose, index) per element
__global__ void pack_kernel(const float* lh, const float* poses, const unsigned* index, long long n,
                            unsigned long long* out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = hsb::best_pack(lh[i], poses + 3 * i, index[i]);
}

// every score of a run of bit patterns with one pose and one index: the packed value, and best_unpack of it
__global__ void pack_sweep_kernel(uint32_t first, long long n, const float* __restrict__ pose, unsigned index,
                                  unsigned long long* packed, float* score, unsigned* index_out) {
  const float p[3] = {pose[0], pose[1], pose[2]};
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long v = hsb::best_pack(arg_of(first, i), p, index);
    unsigned b;
    packed[i] = v;
    score[i] = hsb::best_unpack(v, b);
    index_out[i] = b;
  }
}

struct Dev {
  void* p[8] = {};
  int k = 0;
  cudaError_t err = cudaSuccess;
  void* alloc(size_t bytes) {
    void* q = nullptr;
    if (err == cudaSuccess) err = cudaMalloc(&q, bytes ? bytes : 4);
    p[k++] = q;
    return q;
  }
  void* upload(const void* h, size_t bytes) {
    void* q = alloc(bytes);
    if (err == cudaSuccess && bytes) err = cudaMemcpy(q, h, bytes, cudaMemcpyHostToDevice);
    return q;
  }
  void download(void* h, const void* q, size_t bytes) {
    if (err == cudaSuccess && bytes) err = cudaMemcpy(h, q, bytes, cudaMemcpyDeviceToHost);
  }
  bool ok() const { return err == cudaSuccess; }
  // the launch's own error, then the kernel's
  void launched() {
    if (err == cudaSuccess) err = cudaGetLastError();
    if (err == cudaSuccess) err = cudaDeviceSynchronize();
  }
  ~Dev() {
    for (int i = 0; i < k; ++i) cudaFree(p[i]);
  }
};

unsigned grid_for(long long n) {
  const long long b = (n + 255) / 256;
  return (unsigned)(b < 1 ? 1 : b > 65535 ? 65535 : b);
}

}  // namespace

extern "C" {

// s, c: sinf_glibc, cosf_glibc; ss, sc: the two outputs of sincosf_glibc; n floats each
int hsb_probe_trig_sweep(uint32_t first, long long n, float* s, float* c, float* ss, float* sc) {
  Dev d;
  const size_t b = (size_t)n * 4;
  float *ds = (float*)d.alloc(b), *dc = (float*)d.alloc(b), *dss = (float*)d.alloc(b), *dsc = (float*)d.alloc(b);
  if (!d.ok()) return d.err;
  trig_kernel<<<grid_for(n), 256>>>(first, n, ds, dc, dss, dsc);
  d.launched();
  d.download(s, ds, b); d.download(c, dc, b); d.download(ss, dss, b); d.download(sc, dsc, b);
  return d.err;
}

// e: expf_glibc, n floats
int hsb_probe_exp_sweep(uint32_t first, long long n, float* e) {
  Dev d;
  const size_t b = (size_t)n * 4;
  float* de = (float*)d.alloc(b);
  if (!d.ok()) return d.err;
  exp_kernel<<<grid_for(n), 256>>>(first, n, de);
  d.launched();
  d.download(e, de, b);
  return d.err;
}

// na: normalize_angle, n floats
int hsb_probe_normalize_angle_sweep(uint32_t first, long long n, float* na) {
  Dev d;
  const size_t b = (size_t)n * 4;
  float* dn = (float*)d.alloc(b);
  if (!d.ok()) return d.err;
  norm_sweep_kernel<<<grid_for(n), 256>>>(first, n, dn);
  d.launched();
  d.download(na, dn, b);
  return d.err;
}

int hsb_probe_normalize_angle(const float* in, long long n, float* out) {
  Dev d;
  const size_t b = (size_t)n * 4;
  const float* di = (const float*)d.upload(in, b);
  float* dout = (float*)d.alloc(b);
  if (!d.ok()) return d.err;
  norm_kernel<<<grid_for(n), 256>>>(di, n, dout);
  d.launched();
  d.download(out, dout, b);
  return d.err;
}

int hsb_probe_solve3(const float* h6, const float* d3, long long n, float* out3) {
  Dev d;
  const float* dh = (const float*)d.upload(h6, (size_t)n * 24);
  const float* dd = (const float*)d.upload(d3, (size_t)n * 12);
  float* dout = (float*)d.alloc((size_t)n * 12);
  if (!d.ok()) return d.err;
  solve3_kernel<<<grid_for(n), 256>>>(dh, dd, n, dout);
  d.launched();
  d.download(out3, dout, (size_t)n * 12);
  return d.err;
}

int hsb_probe_pose_difference_larger_than(const float* p1, const float* p2, const float* dist, const float* ang,
                                          long long n, int* out) {
  Dev d;
  const float* d1 = (const float*)d.upload(p1, (size_t)n * 12);
  const float* d2 = (const float*)d.upload(p2, (size_t)n * 12);
  const float* dd = (const float*)d.upload(dist, (size_t)n * 4);
  const float* da = (const float*)d.upload(ang, (size_t)n * 4);
  int* dout = (int*)d.alloc((size_t)n * 4);
  if (!d.ok()) return d.err;
  gate_kernel<<<grid_for(n), 256>>>(d1, d2, dd, da, n, dout);
  d.launched();
  d.download(out, dout, (size_t)n * 4);
  return d.err;
}

int hsb_probe_best_pack(const float* lh, const float* poses, const unsigned* index, long long n, unsigned long long* out) {
  Dev d;
  const float* dl = (const float*)d.upload(lh, (size_t)n * 4);
  const float* dp = (const float*)d.upload(poses, (size_t)n * 12);
  const unsigned* di = (const unsigned*)d.upload(index, (size_t)n * 4);
  unsigned long long* dout = (unsigned long long*)d.alloc((size_t)n * 8);
  if (!d.ok()) return d.err;
  pack_kernel<<<grid_for(n), 256>>>(dl, dp, di, n, dout);
  d.launched();
  d.download(out, dout, (size_t)n * 8);
  return d.err;
}

int hsb_probe_best_pack_sweep(uint32_t first, long long n, const float* pose3, unsigned index, unsigned long long* packed,
                         float* score, unsigned* index_out) {
  Dev d;
  const float* dp = (const float*)d.upload(pose3, 12);
  unsigned long long* dv = (unsigned long long*)d.alloc((size_t)n * 8);
  float* ds = (float*)d.alloc((size_t)n * 4);
  unsigned* di = (unsigned*)d.alloc((size_t)n * 4);
  if (!d.ok()) return d.err;
  pack_sweep_kernel<<<grid_for(n), 256>>>(first, n, dp, index, dv, ds, di);
  d.launched();
  d.download(packed, dv, (size_t)n * 8); d.download(score, ds, (size_t)n * 4); d.download(index_out, di, (size_t)n * 4);
  return d.err;
}

}  // extern "C"
