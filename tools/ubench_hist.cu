// Microbenchmarks that decide the K4 histogram design (build() compiles it to build/ubench_hist).
//  Part A: shared-memory scatter-add throughput per SM for the candidate accumulator schemes
//          (native ATOMS.ADD.32 owner-bank / random-bank, CAS float, non-atomic owner RMW ...).
//  Part B: the engine's K4 kernel (k4_hist_build_ws<4> and <3>, launched through launch_k4) on synthetic
//          tile-major bins: checked exactly against an int64 host computation, then timed with CUDA events
//          and reported as cells/s and algorithmic GB/s.
// Usage: ubench_hist [ROWS] [SKIP_PART_A]   (ROWS defaults to 10M; SKIP_PART_A = 1 skips Part A)
// Output: one JSON document on stdout.  Exit status 1 if the exact check finds a mismatch, except in the
// B200GBM_K4_EXPERIMENT cost-model builds, whose histograms are wrong by design.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <cmath>
#include "../mmlspark_b200/csrc/hist_kernel.cuh"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "CUDA %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1);} } while (0)

using namespace b200gbm;

__device__ __host__ inline unsigned hash32(unsigned x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16; return x;
}

// ---------------------------------------------------------------- Part A
template <int MODE>
__global__ void __launch_bounds__(1024, 1)
ubench(int iters, unsigned long long* cyc_out, unsigned* sink) {
  extern __shared__ __align__(16) unsigned char sm[];
  unsigned* plane = reinterpret_cast<unsigned*>(sm);                  // 4 planes of 8192 words
  unsigned char* sb = sm + 4 * kPlaneWords * 4;                       // 256 rows x 32 B
  int4* sq = reinterpret_cast<int4*>(sb + 256 * 32);                  // 256 rows
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
  for (int e = tid; e < 4 * kPlaneWords; e += blockDim.x) plane[e] = 0;
  for (int e = tid; e < 256 * 32; e += blockDim.x) sb[e] = hash32(e * 2654435761u + blockIdx.x) % 255;
  for (int e = tid; e < 256; e += blockDim.x) sq[e] = make_int4(e - 100, e * 7 + 1, 3, e + 5);
  __syncthreads();
  long long t0 = clock64();
  if (MODE == 9 || MODE == 10) {   // 4 rows x 32 features per warp step, lane = (row selector, bin word), bytes rotated by the row selector; 10 = 3 planes
    const unsigned* sw = reinterpret_cast<const unsigned*>(sb);
    const int rsel = lane >> 3, wsel = lane & 7;
    for (int it = 0; it < iters; ++it) {
#pragma unroll 2
      for (int g4 = warp; g4 < 64; g4 += nwarp) {
        const int r = g4 * 4 + rsel;
        const unsigned word = sw[r * 8 + wsel];
        const int4 q = sq[r];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int kk = (k + rsel) & 3;
          const unsigned b = (word >> (8 * kk)) & 0xFFu;
          const unsigned a = b * 32u + (unsigned)(wsel * 4 + kk);
          atomicAdd(&plane[a], (unsigned)q.x); atomicAdd(&plane[kPlaneWords + a], (unsigned)q.y);
          atomicAdd(&plane[2 * kPlaneWords + a], (unsigned)q.z);
          if (MODE == 9) atomicAdd(&plane[3 * kPlaneWords + a], (unsigned)q.w);
        }
      }
      __syncthreads();
    }
  } else
  for (int it = 0; it < iters; ++it) {
#pragma unroll 4
    for (int r = warp; r < 256; r += nwarp) {
      unsigned b = sb[r * 32 + lane];
      int4 q = sq[r];
      unsigned a = (MODE == 3) ? (lane * 256u + b) : (b * 32u + lane);
      if (MODE == 0 || MODE == 3) {
        atomicAdd(&plane[a], (unsigned)q.x); atomicAdd(&plane[kPlaneWords + a], (unsigned)q.y);
        atomicAdd(&plane[2 * kPlaneWords + a], (unsigned)q.z); atomicAdd(&plane[3 * kPlaneWords + a], (unsigned)q.w);
      } else if (MODE == 1) {
        atomicAdd(&plane[a], (unsigned)q.x); atomicAdd(&plane[kPlaneWords + a], (unsigned)q.y);
      } else if (MODE == 2) {
        atomicAdd(&plane[a], (unsigned)q.x);
      } else if (MODE == 6) {
        atomicAdd(&plane[a], (unsigned)q.x); atomicAdd(&plane[kPlaneWords + a], (unsigned)q.y);
        atomicAdd(&plane[2 * kPlaneWords + a], (unsigned)q.z);
      } else if (MODE == 4) {   // float CAS-loop atomics
        float* fp = reinterpret_cast<float*>(plane);
        atomicAdd(&fp[a], __int_as_float(q.x) * 1e-30f); atomicAdd(&fp[kPlaneWords + a], 1.0f);
      } else if (MODE == 5) {   // non-atomic owner RMW, 64-bit g and h (throughput probe only)
        unsigned long long* p64 = reinterpret_cast<unsigned long long*>(plane);
        unsigned long long g = p64[a], h = p64[kPlaneWords + a];
        p64[a] = g + (unsigned)q.x; p64[kPlaneWords + a] = h + (unsigned)q.y;
      } else if (MODE == 7) {   // loads only
        if (b == 255u && q.x == 123456) plane[a] = 1;
      } else if (MODE == 8) {   // one 64-bit CAS-loop atomic
        unsigned long long* p64 = reinterpret_cast<unsigned long long*>(plane);
        atomicAdd(&p64[a], (unsigned long long)(unsigned)q.x);
      }
    }
    __syncthreads();
  }
  long long t1 = clock64();
  if (tid == 0) cyc_out[blockIdx.x] = (unsigned long long)(t1 - t0);
  unsigned acc = 0;
  for (int e = tid; e < 4 * kPlaneWords; e += blockDim.x) acc += plane[e];
  if (acc == 0xdeadbeef) sink[0] = acc;
}

template <int MODE>
static double run_mode(int threads, int iters, int nsm) {
  unsigned long long* d_cyc; unsigned* d_sink;
  CK(cudaMalloc(&d_cyc, nsm * sizeof(unsigned long long))); CK(cudaMalloc(&d_sink, 4));
  int smem = 4 * kPlaneWords * 4 + 256 * 32 + 256 * 16;
  CK(cudaFuncSetAttribute(ubench<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  ubench<MODE><<<nsm, threads, smem>>>(8, d_cyc, d_sink);
  ubench<MODE><<<nsm, threads, smem>>>(iters, d_cyc, d_sink);
  CK(cudaDeviceSynchronize());
  std::vector<unsigned long long> c(nsm);
  CK(cudaMemcpy(c.data(), d_cyc, nsm * 8, cudaMemcpyDeviceToHost));
  double s = 0; for (auto v : c) s += (double)v;
  s /= nsm;
  CK(cudaFree(d_cyc)); CK(cudaFree(d_sink));
  return (double)iters * 256.0 * 32.0 / s;   // cells per cycle per SM
}

// ---------------------------------------------------------------- Part B
__global__ void gen_bins(uint8_t* bins, size_t rows_stride, int num_tiles, size_t n, unsigned seed) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;   // one 4-byte word each
  size_t total = (size_t)num_tiles * rows_stride * 8;
  for (; i < total; i += (size_t)gridDim.x * blockDim.x) {
    unsigned w = 0;
    for (int k = 0; k < 4; ++k) w |= (hash32((unsigned)(i * 4 + k) ^ seed) % 255u) << (8 * k);
    reinterpret_cast<unsigned*>(bins)[i] = w;
  }
}
__global__ void gen_q(int4* q, size_t n, unsigned seed) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  for (; i < n; i += (size_t)gridDim.x * blockDim.x) {
    long long g = (long long)(int)hash32((unsigned)i ^ seed) * 11LL;                 // signed ~36 bit
    long long h = (long long)(hash32((unsigned)i * 3u + seed) >> 1) * 9LL;           // unsigned ~35 bit
    q[i] = make_int4((int)(g >> kLoBits), (int)(g & ((1 << kLoBits) - 1)), (int)(h >> kLoBits), (int)(h & ((1 << kLoBits) - 1)));
  }
}
__global__ void gen_idx(int* idx, int n, int stride) {   // every `stride`-th row, ascending
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  for (; i < n; i += gridDim.x * blockDim.x) idx[i] = i * stride;
}

int main(int argc, char** argv) {
  int dev = 0; CK(cudaSetDevice(dev));
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, dev));
  int nsm = prop.multiProcessorCount;
  printf("{\n \"gpu\": \"%s\", \"sms\": %d, \"clock_khz\": %d,\n", prop.name, nsm, prop.clockRate);

  // ---- Part A
  printf(" \"smem_scatter_cells_per_cycle_per_sm\": {\n");
  const int it = 400;
  for (int threads : {512, 1024}) {
    if (argc > 2 && atoi(argv[2]) == 1) { printf("  \"t%d\": {}%s\n", threads, threads == 512 ? "," : ""); continue; }
    printf("  \"t%d\": {", threads);
    printf("\"u32x4_rows4x32_rotated\": %.3f, ", run_mode<9>(threads, it, nsm));
    printf("\"u32x3_rows4x32_rotated\": %.3f, ", run_mode<10>(threads, it, nsm));
    printf("\"u32x4_ownerbank\": %.3f, ", run_mode<0>(threads, it, nsm));
    printf("\"u32x3_ownerbank\": %.3f, ", run_mode<6>(threads, it, nsm));
    printf("\"u32x2_ownerbank\": %.3f, ", run_mode<1>(threads, it, nsm));
    printf("\"u32x1_ownerbank\": %.3f, ", run_mode<2>(threads, it, nsm));
    printf("\"u32x4_randombank\": %.3f, ", run_mode<3>(threads, it, nsm));
    printf("\"f32x2_cas_ownerbank\": %.3f, ", run_mode<4>(threads, it / 4, nsm));
    printf("\"u64x2_nonatomic_rmw\": %.3f, ", run_mode<5>(threads, it, nsm));
    printf("\"u64x1_cas\": %.3f, ", run_mode<8>(threads, it / 4, nsm));
    printf("\"loads_only\": %.3f}%s\n", run_mode<7>(threads, it, nsm), threads == 512 ? "," : "");
  }
  printf(" },\n");

  if (const char* e = getenv("B200GBM_L2_FETCH")) {
    CK(cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)atoi(e)));
  }
  { size_t g = 0; cudaDeviceGetLimit(&g, cudaLimitMaxL2FetchGranularity); printf(" \"l2_fetch_granularity\": %zu,\n", g); }
  // ---- Part B
  const int F = 256, num_tiles = F / 32;
  size_t N = (argc > 1) ? (size_t)atoll(argv[1]) : 10000000;
  size_t rows_stride = (N + 255) / 256 * 256;
  uint8_t* d_bins; int4* d_q; int4* d_qord; int* d_idx; unsigned long long* d_hist; HistWork* d_work;
  size_t slot_elems = (size_t)F * 256 * 2;
  CK(cudaMalloc(&d_bins, (size_t)num_tiles * rows_stride * 32));
  CK(cudaMalloc(&d_q, N * sizeof(int4)));
  CK(cudaMalloc(&d_qord, N * sizeof(int4)));
  CK(cudaMalloc(&d_idx, N * sizeof(int)));
  CK(cudaMalloc(&d_hist, slot_elems * 8));
  CK(cudaMalloc(&d_work, sizeof(HistWork) * 2));
  gen_bins<<<nsm * 8, 256>>>(d_bins, rows_stride, num_tiles, N, 12345u);
  gen_q<<<nsm * 8, 256>>>(d_q, N, 777u);
  CK(cudaDeviceSynchronize());
  CK(set_k4_smem_limit());

  // exact int64 check of both instantiations on the first 1M rows: a contiguous pass and a strided index-list pass (every 3rd
  // row), each with CTAs sharing feature tiles.  NATOM = 3 sums the count field q.z as h, as the kernel does.
  size_t k4_bad = 0;
  {
    const int n_chk = (int)std::min<size_t>(N, 1000000);
    HistWork hw[2] = {{0, n_chk, 0, 0}, {0, n_chk / 3, 1, 0}};
    CK(cudaMemcpy(d_work, hw, sizeof(hw), cudaMemcpyHostToDevice));
    gen_idx<<<nsm, 256>>>(d_idx, n_chk / 3, 3);
    k_gather_q<<<nsm * 8, 256>>>(d_work + 1, d_idx, d_idx, d_q, d_qord);
    CK(cudaDeviceSynchronize());
    std::vector<uint8_t> hb((size_t)num_tiles * rows_stride * 32);
    CK(cudaMemcpy(hb.data(), d_bins, hb.size(), cudaMemcpyDeviceToHost));
    std::vector<int4> hq(n_chk);
    CK(cudaMemcpy(hq.data(), d_q, (size_t)n_chk * 16, cudaMemcpyDeviceToHost));
    std::vector<long long> got(slot_elems), want(slot_elems);
    printf(" \"k4_check\": {\"rows\": %d, \"mismatches\": {", n_chk);
    for (int natom : {4, 3}) {
      for (int pass = 0; pass < 2; ++pass) {
        CK(cudaMemset(d_hist, 0, slot_elems * 8));
        launch_k4(natom == 3, d_bins, rows_stride, num_tiles, d_q, d_qord, d_idx, d_idx, d_work + pass, d_hist, nsm, 0);
        CK(cudaGetLastError());
        CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(got.data(), d_hist, slot_elems * 8, cudaMemcpyDeviceToHost));
        std::fill(want.begin(), want.end(), 0LL);
        const int step = pass ? 3 : 1;
        for (int i = 0; i < hw[pass].count * step; i += step) {
          const long long g = ((long long)hq[i].x << kLoBits) + hq[i].y;
          const long long h = natom == 4 ? ((long long)hq[i].z << kLoBits) + hq[i].w : (long long)hq[i].z;
          for (int t = 0; t < num_tiles; ++t) {
            const uint8_t* row = &hb[((size_t)t * rows_stride + i) * 32];
            for (int l = 0; l < 32; ++l) {
              size_t o = ((size_t)(t * 32 + l) * 256 + row[l]) * 2;
              want[o] += g; want[o + 1] += h;
            }
          }
        }
        size_t bad = 0; for (size_t i = 0; i < want.size(); ++i) bad += (got[i] != want[i]);
        printf("%s\"natom%d_%s\": %zu", natom == 4 && pass == 0 ? "" : ", ", natom, pass ? "gathered" : "contiguous", bad);
        k4_bad += bad;
      }
    }
    printf("}},\n");
  }

  // timing: full pass (contiguous) and gathered pass (every 2nd row), NATOM 4 and 3
  auto time_it = [&](int natom, int n, int use_idx, int reps) -> float {
    HistWork hw = {0, n, use_idx, 0};
    CK(cudaMemcpy(d_work, &hw, sizeof(hw), cudaMemcpyHostToDevice));
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    float best = 1e30f, tot = 0;
    for (int r = 0; r < reps + 2; ++r) {
      CK(cudaMemsetAsync(d_hist, 0, slot_elems * 8));
      CK(cudaEventRecord(e0));
      if (use_idx) k_gather_q<<<nsm * 8, 256>>>(d_work, d_idx, d_idx, d_q, d_qord);     // part of a leaf pass: timed
      launch_k4(natom == 3, d_bins, rows_stride, num_tiles, d_q, d_qord, d_idx, d_idx, d_work, d_hist, nsm, 0);
      CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
      if (r >= 2) { best = std::min(best, ms); tot += ms; }
    }
    (void)best;
    return tot / reps;
  };
  printf(" \"k4_timing\": [\n");
  struct Cfg { int natom; double frac; int use_idx; };
  Cfg cfgs[] = {{4, 1.0, 0}, {3, 1.0, 0}, {4, 0.5, 1}, {4, 0.1, 1}, {4, 0.01, 1}, {4, 0.001, 1}};
  for (size_t c = 0; c < sizeof(cfgs) / sizeof(cfgs[0]); ++c) {
    int n = (int)(N * cfgs[c].frac);
    if (cfgs[c].use_idx) { gen_idx<<<nsm, 256>>>(d_idx, n, (int)(1.0 / cfgs[c].frac)); CK(cudaDeviceSynchronize()); }
    float ms = time_it(cfgs[c].natom, n, cfgs[c].use_idx, 5);
    double cells = (double)n * F;
    double bytes = (double)n * (F + 16.0 * num_tiles + (cfgs[c].use_idx ? 4.0 * num_tiles : 0.0)) + (double)F * 256 * 16;
    printf("  {\"natom\": %d, \"rows\": %d, \"gather\": %d, \"ms\": %.4f, \"gcells_per_s\": %.2f, \"algo_GBps\": %.1f}%s\n",
           cfgs[c].natom, n, cfgs[c].use_idx, ms, cells / ms * 1e-6, bytes / ms * 1e-6, c + 1 < sizeof(cfgs) / sizeof(cfgs[0]) ? "," : "");
  }
  printf(" ]\n}\n");
  return (B200GBM_K4_EXPERIMENT == 0 && k4_bad != 0) ? 1 : 0;
}
