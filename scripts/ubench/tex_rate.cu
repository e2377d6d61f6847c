// Diagnostic: what does one warp-level texture gather cost an SM, by texel format and by how the 32 lanes'
// footprints are spread?  K1 (match_kernel) issues one warp-level TLD4 per 32 unrelated 2x2 footprints; this probe
// separates the pipe's own rate (all lanes on one footprint) from the cost of
// divergence, and measures the alternatives that would return the same four fp32 values per endpoint:
//   tld4      tld4.r.2d on an R32F array            (4 texels of a 2x2 footprint, what K1 issues)
//   rgba      tex.2d.v4 on an RGBA32F array         (ONE 16-byte texel = a pre-packed neighbourhood)
//   rg x2     2 x tex.2d on an RG32F array          (two 8-byte texels: rows y and y+1 of a pair plane)
//   r x1      tex.2d on an R32F array, one value    (the pipe's rate for a 1-register return)
//   ldg128    ld.global.v4 from a linear float4 plane (the LSU path with the same packed neighbourhood)
//   ldg64x2   2 x ld.global.v2 from a pair plane;  ldg32x4: 4 x ld.global.f32 from the plain plane (K1's MODE_LDG)
//   tld4+128 / tld4+64: every other gather through the texture path, the others through the LSU path — do they overlap?
// Output: ns and SM cycles (at the clock measured in the kernel) per warp-level gather per SM, 28 warps per SM.
// `resident`: each warp keeps coming back to a fixed set of scan-like footprints; sweeps the per-SM working set,
// warps per SM and the L1 size (a K1-sized shared-memory request against none) — what an L1 hit saves a scan gather.
// Build: make -C scripts/ubench bin/tex_rate     Run: bin/tex_rate [resident] [map size, default 2048]
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1);} } while (0)

enum Op { OP_TLD4 = 0, OP_RGBA = 1, OP_RG2 = 2, OP_R1 = 3, OP_LDG128 = 4, OP_LDG64X2 = 5, OP_LDG32X4 = 6, OP_MIX128 = 7, OP_MIX64 = 8 };
enum Pattern { PAT_SAME = 0, PAT_CONSEC = 1, PAT_WINDOW = 2, PAT_RANDOM = 3, PAT_SCAN = 4 };

struct Args {
  cudaTextureObject_t tex;
  const float4* plane;   // OP_LDG128
  int size, mask, iters, pattern;
  float* out;
  unsigned long long* clocks;   // per block: elapsed clock64 of warp 0
};

__device__ __forceinline__ float u2f(unsigned v) { return __uint_as_float(0x4B000000u | v) - 8388608.0f; }   // exact for v < 2^23

template <int OP>
__device__ __forceinline__ float gather(const Args& A, float x, float y) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (OP == OP_TLD4) {
    asm volatile("tld4.r.2d.v4.f32.f32 {%0,%1,%2,%3}, [%4, {%5,%6}];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(A.tex), "f"(x), "f"(y));
  } else if (OP == OP_RGBA) {
    asm volatile("tex.2d.v4.f32.f32 {%0,%1,%2,%3}, [%4, {%5,%6}];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(A.tex), "f"(x), "f"(y));
  } else if (OP == OP_RG2) {
    float a, b, c, d, t0, t1;
    asm volatile("tex.2d.v4.f32.f32 {%0,%1,%2,%3}, [%4, {%5,%6}];" : "=f"(a), "=f"(b), "=f"(t0), "=f"(t1) : "l"(A.tex), "f"(x), "f"(y));
    asm volatile("tex.2d.v4.f32.f32 {%0,%1,%2,%3}, [%4, {%5,%6}];" : "=f"(c), "=f"(d), "=f"(t0), "=f"(t1) : "l"(A.tex), "f"(x), "f"(y + 1.0f));
    v = make_float4(a, b, c, d);
  } else if (OP == OP_R1) {
    float t0, t1, t2;
    asm volatile("tex.2d.v4.f32.f32 {%0,%1,%2,%3}, [%4, {%5,%6}];" : "=f"(v.x), "=f"(t0), "=f"(t1), "=f"(t2) : "l"(A.tex), "f"(x), "f"(y));
  } else if (OP == OP_LDG128) {
    const int ix = (int)x, iy = (int)y;
    v = __ldg(A.plane + (size_t)iy * A.size + ix);
  } else if (OP == OP_LDG64X2) {   // pair plane: {P(x,y), P(x+1,y)} per cell, rows y and y+1
    const int ix = (int)x, iy = (int)y;
    const float2* pl = reinterpret_cast<const float2*>(A.plane);
    const float2 a = __ldg(pl + (size_t)iy * A.size + ix), b = __ldg(pl + (size_t)(iy + 1) * A.size + ix);
    v = make_float4(a.x, a.y, b.x, b.y);
  } else {   // OP_LDG32X4: the plain plane, four scalar loads (K1's MODE_LDG)
    const int ix = (int)x, iy = (int)y;
    const float* pl = reinterpret_cast<const float*>(A.plane);
    const float* r0 = pl + (size_t)iy * A.size + ix;
    v = make_float4(__ldg(r0), __ldg(r0 + 1), __ldg(r0 + A.size), __ldg(r0 + A.size + 1));
  }
  return (v.x + v.y) + (v.z + v.w);
}
// mixes: gathers alternate between the texture path and the load/store path — do the two overlap?
template <int OP, int u>
__device__ __forceinline__ float gather_mix(const Args& A, float x, float y) {
  if (OP == OP_MIX128) return (u & 1) ? gather<OP_LDG128>(A, x, y) : gather<OP_TLD4>(A, x, y);
  if (OP == OP_MIX64) return (u & 1) ? gather<OP_LDG64X2>(A, x, y) : gather<OP_TLD4>(A, x, y);
  return gather<OP>(A, x, y);
}

template <int OP, int U>
__global__ void __launch_bounds__(896, 1) rate_kernel(const Args A) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned s = (blockIdx.x * 977u + warp * 131u + 7u) * 2654435761u;          // warp-uniform stream
  unsigned sl = s ^ (lane * 0x9E3779B9u);                                       // per-lane stream
  float acc = 0.f;
  const unsigned m = (unsigned)A.mask;
  const long long c0 = clock64();
  for (int it = 0; it < A.iters; ++it) {
    float xs[U], ys[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      s = s * 1664525u + 1013904223u;
      sl = sl * 1664525u + 1013904223u;
      const unsigned bx = (s >> 7) & m, by = (s >> 19) & m;
      unsigned x, y;
      if (A.pattern == PAT_SAME) { x = bx; y = by; }
      else if (A.pattern == PAT_CONSEC) { x = (bx + lane) & m; y = by; }
      else if (A.pattern == PAT_WINDOW) { x = (bx + ((sl >> 9) & 63u)) & m; y = (by + ((sl >> 21) & 63u)) & m; }
      else if (A.pattern == PAT_RANDOM) { x = (sl >> 7) & m; y = (sl >> 19) & m; }
      else {   // scan-like: consecutive beams hit a wall 1.5 cells apart along a direction that changes per gather
        const unsigned dir = (s >> 3) & 3u;
        const unsigned step = (lane * 3u) >> 1;
        x = (bx + ((dir & 1u) ? step : (lane >> 3))) & m;
        y = (by + ((dir & 1u) ? (lane >> 3) : step)) & m;
      }
      if (x >= m) x = m - 1;   // keep the 2x2 footprint inside
      if (y >= m) y = m - 1;
      xs[u] = u2f(x);
      ys[u] = u2f(y);
    }
    float r[U];
#pragma unroll
    for (int u = 0; u < U; ++u) r[u] = (u & 1) ? gather_mix<OP, 1>(A, xs[u], ys[u]) : gather_mix<OP, 0>(A, xs[u], ys[u]);
#pragma unroll
    for (int u = 0; u < U; ++u) acc += r[u];
  }
  const long long c1 = clock64();
  if (acc == 123.456f) A.out[0] = acc;   // keep the gathers alive
  if (threadIdx.x == 0) A.clocks[blockIdx.x] = (unsigned long long)(c1 - c0);
}

// Resident footprints: warp w of an SM cycles through F scan-like footprints of its own (the "scan" pattern's shape,
// bases drawn once per footprint), so from the second pass on every gather finds its cells in L1 when the SM's
// working set (warps x F footprints) fits there.  F at least the number of gathers a warp issues = every footprint
// new, the "scan" pattern under the same code.  The dynamic shared-memory request only sets the carve-out.
template <int U>
__global__ void __launch_bounds__(1024, 1) resident_kernel(const Args A, int F) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned seed = (blockIdx.x * 977u + warp * 131u + 7u) * 2654435761u;
  const unsigned m = (unsigned)A.mask;
  const unsigned step = (lane * 3u) >> 1, row = (unsigned)lane >> 3;
  float acc = 0.f;
  int k = 0;
  const long long c0 = clock64();
  for (int it = 0; it < A.iters; ++it) {
    float xs[U], ys[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned s = (seed ^ ((unsigned)k * 0x9E3779B9u)) * 1664525u + 1013904223u;
      const unsigned bx = (s >> 7) & m, by = (s >> 19) & m, dir = (s >> 3) & 1u;
      unsigned x = (bx + (dir ? step : row)) & m, y = (by + (dir ? row : step)) & m;
      if (x >= m) x = m - 1;
      if (y >= m) y = m - 1;
      xs[u] = u2f(x);
      ys[u] = u2f(y);
      k = (k + 1 == F) ? 0 : k + 1;
    }
    float r[U];
#pragma unroll
    for (int u = 0; u < U; ++u) r[u] = gather<OP_TLD4>(A, xs[u], ys[u]);
#pragma unroll
    for (int u = 0; u < U; ++u) acc += r[u];
  }
  const long long c1 = clock64();
  if (acc == 123.456f) A.out[0] = acc;
  if (threadIdx.x == 0) A.clocks[blockIdx.x] = (unsigned long long)(c1 - c0);
}

// Cycles per warp-level tld4 per SM for resident footprints, against L1 size (dynamic shared memory request) x
// warps per SM x per-SM working set.  A footprint is counted as 16 sectors (512 B): lanes 1.5 cells apart on 4 rows
// of a 2x2 footprint each, ~100 distinct fp32 cells in a block-linear layout.
static void resident_sweep(Args A, int sms) {
  constexpr int U = 4;
  constexpr int kFootprintBytes = 512;
  const int big_smem = 227 * 1024;   // leaves 28 KB of the 256 KB for L1, as a fully staged one-wave K1 CTA does
  CK(cudaFuncSetAttribute(resident_kernel<U>, cudaFuncAttributeMaxDynamicSharedMemorySize, big_smem));
  std::vector<unsigned long long> clk(sms);
  const int warps_list[4] = {8, 16, 28, 32};
  const int ws_kb[5] = {16, 64, 128, 480, 0};   // 0: no reuse (every footprint new)
  printf("resident tld4 footprints: cycles per warp-level gather per SM (%d SMs, %d gathers per warp)\n", sms, A.iters * U);
  for (int cfg = 0; cfg < 2; ++cfg) {
    const int smem = cfg == 0 ? big_smem : 0;
    CK(cudaFuncSetAttribute(resident_kernel<U>, cudaFuncAttributePreferredSharedMemoryCarveout, cfg == 0 ? 100 : 0));
    printf("%s\n", cfg == 0 ? "L1 ~28 KB (227 KB dynamic shared memory)" : "L1 maximal (no shared memory, carve-out 0)");
    printf("  warps/SM");
    for (int w : ws_kb) w ? printf("  %6d KB", w) : printf("  no reuse");
    printf("   no-reuse / best\n");
    for (int warps : warps_list) {
      printf("  %8d", warps);
      double best = 1e30, none = 0;
      for (int w : ws_kb) {
        const int F = w ? std::max(1, (w * 1024) / (warps * kFootprintBytes)) : A.iters * U;
        resident_kernel<U><<<sms, warps * 32, smem>>>(A, F);
        CK(cudaGetLastError());
        CK(cudaDeviceSynchronize());
        resident_kernel<U><<<sms, warps * 32, smem>>>(A, F);
        CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(clk.data(), A.clocks, sizeof(unsigned long long) * sms, cudaMemcpyDeviceToHost));
        double cyc = 0;
        for (int i = 0; i < sms; ++i) cyc += (double)clk[i];
        cyc /= (double)sms * A.iters * U * warps;
        printf("  %9.2f", cyc);
        if (w) best = std::min(best, cyc); else none = cyc;
      }
      printf("   %6.2fx\n", none / best);
    }
  }
}

template <int OP>
static void run(const char* name, Args A, int sms, int warps, const char* const* pat_names) {
  constexpr int U = 4;
  std::vector<unsigned long long> clk(sms);
  printf("%-8s", name);
  for (int pat = 0; pat < 5; ++pat) {
    A.pattern = pat;
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    rate_kernel<OP, U><<<sms, warps * 32>>>(A);
    CK(cudaDeviceSynchronize());
    CK(cudaEventRecord(e0));
    rate_kernel<OP, U><<<sms, warps * 32>>>(A);
    CK(cudaEventRecord(e1));
    CK(cudaDeviceSynchronize());
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    CK(cudaMemcpy(clk.data(), A.clocks, sizeof(unsigned long long) * sms, cudaMemcpyDeviceToHost));
    double cyc = 0;
    for (int i = 0; i < sms; ++i) cyc += (double)clk[i];
    cyc /= sms;
    const double gathers_per_sm = (double)A.iters * U * warps;
    printf("  %s %6.2f cyc (%5.2f ns)", pat_names[pat], cyc / gathers_per_sm, ms * 1e6 / gathers_per_sm);
    (void)pat_names;
  }
  printf("\n");
}

int main(int argc, char** argv) {
  const bool resident = argc > 1 && strcmp(argv[1], "resident") == 0;
  if (resident) { --argc; ++argv; }
  const int size = argc > 1 ? atoi(argv[1]) : 2048;
  const int warps = argc > 2 ? atoi(argv[2]) : 28;
  int dev = 0, sms = 0;
  CK(cudaGetDevice(&dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  printf("map %d^2, %d SMs, %d warps per SM, 4 gathers in flight per lane; cost per WARP-level gather per SM\n", size, sms, warps);
  std::vector<float> h((size_t)size * size * 4);
  unsigned s = 12345u;
  for (auto& v : h) { s = s * 1664525u + 1013904223u; v = (float)(s >> 8) * (1.0f / 16777216.0f); }

  auto make_tex = [&](int channels, cudaArray_t* arr_out) {
    cudaChannelFormatDesc d = channels == 1 ? cudaCreateChannelDesc<float>() : channels == 2 ? cudaCreateChannelDesc<float2>() : cudaCreateChannelDesc<float4>();
    cudaArray_t arr;
    CK(cudaMallocArray(&arr, &d, size, size));
    CK(cudaMemcpy2DToArray(arr, 0, 0, h.data(), (size_t)size * channels * 4, (size_t)size * channels * 4, size, cudaMemcpyHostToDevice));
    cudaResourceDesc rd = {};
    rd.resType = cudaResourceTypeArray;
    rd.res.array.array = arr;
    cudaTextureDesc td = {};
    td.addressMode[0] = td.addressMode[1] = cudaAddressModeClamp;
    td.filterMode = cudaFilterModePoint;
    td.readMode = cudaReadModeElementType;
    td.normalizedCoords = 0;
    cudaTextureObject_t t;
    CK(cudaCreateTextureObject(&t, &rd, &td, nullptr));
    *arr_out = arr;
    return t;
  };
  cudaArray_t a1, a2, a4;
  cudaTextureObject_t t1 = make_tex(1, &a1), t2 = make_tex(2, &a2), t4 = make_tex(4, &a4);
  float4* plane;
  CK(cudaMalloc(&plane, (size_t)size * size * 16));
  CK(cudaMemcpy(plane, h.data(), (size_t)size * size * 16, cudaMemcpyHostToDevice));
  Args A = {};
  A.size = size;
  A.mask = size - 1;
  A.iters = 2000;
  A.plane = plane;
  CK(cudaMalloc(&A.out, 16));
  CK(cudaMalloc(&A.clocks, sizeof(unsigned long long) * sms));
  const char* pats[5] = {"same", "consec", "win64", "random", "scan"};
  if (resident) {
    A.tex = t1;
    resident_sweep(A, sms);
    return 0;
  }
  A.tex = t1;
  run<OP_TLD4>("tld4", A, sms, warps, pats);
  A.tex = t4;
  run<OP_RGBA>("rgba", A, sms, warps, pats);
  A.tex = t2;
  run<OP_RG2>("rg x2", A, sms, warps, pats);
  A.tex = t1;
  run<OP_R1>("r x1", A, sms, warps, pats);
  run<OP_LDG128>("ldg128", A, sms, warps, pats);
  run<OP_LDG64X2>("ldg64x2", A, sms, warps, pats);
  run<OP_LDG32X4>("ldg32x4", A, sms, warps, pats);
  run<OP_MIX128>("tld4+128", A, sms, warps, pats);
  run<OP_MIX64>("tld4+64", A, sms, warps, pats);
  return 0;
}
