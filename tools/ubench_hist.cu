// Microbenchmarks that decide the K4 histogram design (build() compiles it to build/ubench_hist).
//  Part A: shared-memory scatter-add throughput per SM for the candidate accumulator schemes
//          (native ATOMS.ADD.32 owner-bank / random-bank, CAS float, non-atomic owner RMW ...).
//  Part B: the engine's K4 kernel (k4_hist_build_ws<4> and <3>, and quantised training's packed k4_hist_build_packed, with and
//          without the count plane, all launched through launch_k4 with the per-block bin-count
//          bound of launch_block_bound) on synthetic tile-major bins, uniform and skewed: checked exactly against an int64
//          host computation, then timed with CUDA events and reported as cells/s and algorithmic GB/s.
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
// (g,h) words with signed ~36-bit g and unsigned ~35-bit h whose 18-bit low fields lie in [2^18 - 2^12, 2^18): one cell's low
// field fits 2^14 additions and wraps its 32-bit accumulator within ~16.6K, so a window that misses a needed flush gives a mismatch
__global__ void gen_q(int4* q, size_t n, unsigned seed) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  for (; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int g_hi = (int)hash32((unsigned)i ^ seed) >> 14, h_hi = (int)(hash32((unsigned)i * 3u + seed) >> 15);
    const int g_lo = (1 << kLoBits) - 1 - (int)(hash32((unsigned)i * 5u + seed) & 4095u);
    const int h_lo = (1 << kLoBits) - 1 - (int)(hash32((unsigned)i * 7u + seed) & 4095u);
    q[i] = make_int4(g_hi, g_lo, h_hi, h_lo);
  }
}
// quantised (g,h) words of the packed instantiation, in K3's layout: q_g = +-floor(B/2) and q_h = +-B (1 in 8 negative), the field
// limits, so that a cell that takes more than packed_flush_cap additions between flushes leaves its 16-bit field and mismatches
__global__ void gen_q_packed(int4* q, size_t n, int B, unsigned seed) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  for (; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int qg = (hash32((unsigned)i ^ seed) & 7u) ? B / 2 : -(B / 2), qh = (hash32((unsigned)i * 3u + seed) & 7u) ? B : -B;
    q[i] = make_int4(qg >> kLoBits, qg & ((1 << kLoBits) - 1), qh >> kLoBits, qh & ((1 << kLoBits) - 1));
  }
}
__global__ void gen_idx(int* idx, int n, int stride) {   // every `stride`-th row, ascending
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  for (; i < n; i += gridDim.x * blockDim.x) idx[i] = i * stride;
}
// skew: column `col` of `tile` takes bin 7 in every row of [r0, r1) except every 64th, so one cell collects far more than 2^14
// rows of a CTA's range and the flush bound has to force flushes
__global__ void skew_bins(uint8_t* bins, size_t rows_stride, int tile, int col, int r0, int r1) {
  for (int r = r0 + blockIdx.x * blockDim.x + threadIdx.x; r < r1; r += gridDim.x * blockDim.x)
    if (r % 64 != 0) bins[((size_t)tile * rows_stride + r) * 32 + col] = 7;
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
  int4* d_qp; CK(cudaMalloc(&d_qp, N * sizeof(int4)));      // the packed instantiation's words (gen_q_packed)
  CK(cudaMalloc(&d_qord, 2 * N * sizeof(int4)));      // the second half: the packed words in leaf order (k4_check)
  CK(cudaMalloc(&d_idx, N * sizeof(int)));
  CK(cudaMalloc(&d_hist, slot_elems * 8));
  CK(cudaMalloc(&d_work, sizeof(HistWork) * 2));
  // the per-block bin-count bound of the flush rule, computed by the engine's kernels whenever the bins change
  int* d_bound; CK(cudaMalloc(&d_bound, sizeof(int) * num_tiles * (bound_blocks((int)N) + 1)));
  const RowBlockBound kb{d_bound, bound_blocks((int)N)};
  auto set_bins = [&](int skew_r0, int skew_r1) {      // uniform bins, optionally skewed in rows [skew_r0, skew_r1), and their bound
    gen_bins<<<nsm * 8, 256>>>(d_bins, rows_stride, num_tiles, N, 12345u);
    if (skew_r1 > skew_r0) skew_bins<<<nsm * 8, 256>>>(d_bins, rows_stride, 1, 5, skew_r0, skew_r1);
    launch_block_bound(d_bins, rows_stride, (int)N, num_tiles, F, d_bound, 0);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
  };
  gen_q<<<nsm * 8, 256>>>(d_q, N, 777u);
  // kinds of K4 launch: NATOM 4 and 3 on d_q; packed (quantised training) on d_qp at kPackedB, with the words' q_h ("packed") or
  // q_h = 1 ("packed_count")
  const int kPackedB = 63;      // the largest B: the smallest cap (520 additions), so the flush rule is tested hardest
  gen_q_packed<<<nsm * 8, 256>>>(d_qp, N, kPackedB, 999u);
  enum Kind { kN4, kN3, kPacked, kPackedCount };
  const char* kind_name[] = {"natom4", "natom3", "packed", "packed_count"};
  auto launch = [&](Kind k, int quant_bins, int4* qord, RowBlockBound rb) {
    const bool packed = k == kPacked || k == kPackedCount;
    launch_k4(k == kN3 || k == kPackedCount, packed ? quant_bins : 0, d_bins, rows_stride, num_tiles, packed ? d_qp : d_q, qord, d_idx, d_idx,
              d_work, d_hist, rb, nsm, 0);
  };
  set_bins(0, 0);
  CK(set_k4_smem_limit());

  // exact int64 check of both instantiations on the first 1M rows, every pass with CTAs sharing feature tiles: a contiguous pass
  // and an ascending index-list pass, on three bin states.  "uniform": the generated bins, every 3rd row gathered.  "skew": column 5
  // of tile 1 has nearly every row in one bin, so the bound must force flushes; every 2nd row gathered.  "skew_second_half": the
  // same skew in the second half of the rows only, so a window that starts uniform must flush in time; every 37th row gathered (a
  // leaf of low density).  NATOM = 3 sums the count field q.z as h, as the kernel does.
  size_t k4_bad = 0;
  {
    const int n_chk = (int)std::min<size_t>(N, 1000000);
    std::vector<uint8_t> hb((size_t)num_tiles * n_chk * 32);      // [tile][row][32] of the checked rows
    std::vector<int4> hq(n_chk), hqp(n_chk);
    CK(cudaMemcpy(hq.data(), d_q, (size_t)n_chk * 16, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(hqp.data(), d_qp, (size_t)n_chk * 16, cudaMemcpyDeviceToHost));
    std::vector<long long> got(slot_elems), want[4];
    for (auto& v : want) v.resize(slot_elems);
    printf(" \"k4_check\": {\"rows\": %d, \"mismatches\": {", n_chk);
    struct State { const char* name; int skew_r0, skew_r1, stride; };
    const State states[] = {{"uniform", 0, 0, 3}, {"skew", 0, n_chk, 2}, {"skew_second_half", n_chk / 2, n_chk, 37}};
    bool first = true;
    for (const State& st : states) {
      set_bins(st.skew_r0, st.skew_r1);
      for (int t = 0; t < num_tiles; ++t)
        CK(cudaMemcpy(&hb[(size_t)t * n_chk * 32], d_bins + (size_t)t * rows_stride * 32, (size_t)n_chk * 32, cudaMemcpyDeviceToHost));
      for (int pass = 0; pass < 2; ++pass) {
        const int step = pass ? st.stride : 1;
        const HistWork hw = {0, n_chk / step, pass, 0};
        CK(cudaMemcpy(d_work, &hw, sizeof(hw), cudaMemcpyHostToDevice));
        int4* d_qpord = d_qord + n_chk;      // the packed words in leaf order, beside d_q's
        if (pass) {
          gen_idx<<<nsm, 256>>>(d_idx, hw.count, step);
          k_gather_q<<<nsm * 8, 256>>>(d_work, d_idx, d_idx, d_q, d_qord);
          k_gather_q<<<nsm * 8, 256>>>(d_work, d_idx, d_idx, d_qp, d_qpord);
        }
        for (auto& v : want) std::fill(v.begin(), v.end(), 0LL);
        for (int i = 0; i < hw.count * step; i += step) {
          const long long g = ((long long)hq[i].x << kLoBits) + hq[i].y;
          const long long gp = ((long long)hqp[i].x << kLoBits) + hqp[i].y, hp = ((long long)hqp[i].z << kLoBits) + hqp[i].w;
          const long long gh[4][2] = {{g, ((long long)hq[i].z << kLoBits) + hq[i].w}, {g, hq[i].z}, {gp, hp}, {gp, 1}};
          for (int t = 0; t < num_tiles; ++t) {
            const uint8_t* row = &hb[((size_t)t * n_chk + i) * 32];
            for (int l = 0; l < 32; ++l) {
              size_t o = ((size_t)(t * 32 + l) * 256 + row[l]) * 2;
              for (int k = 0; k < 4; ++k) { want[k][o] += gh[k][0]; want[k][o + 1] += gh[k][1]; }
            }
          }
        }
        for (Kind k : {kN4, kN3, kPacked, kPackedCount}) {
          CK(cudaMemset(d_hist, 0, slot_elems * 8));
          launch(k, kPackedB, (k == kPacked || k == kPackedCount) ? d_qpord : d_qord, kb);
          CK(cudaGetLastError());
          CK(cudaDeviceSynchronize());
          CK(cudaMemcpy(got.data(), d_hist, slot_elems * 8, cudaMemcpyDeviceToHost));
          size_t bad = 0; for (size_t i = 0; i < slot_elems; ++i) bad += (got[i] != want[k][i]);
          printf("%s\"%s_%s_%s\": %zu", first ? "" : ", ", st.name, kind_name[k], pass ? "gathered" : "contiguous", bad);
          first = false;
          k4_bad += bad;
        }
      }
    }
    printf("}},\n");
    set_bins(0, 0);
  }

  // timing: full pass (contiguous) and gathered passes, NATOM 4 and 3.  The two skew = 1 rows run on bins whose column 5 of tile 1
  // has nearly every row in one bin, where the block bound lets that tile flush only every ~2^14 rows: once with the block bound
  // and once (bound = 0) with the row-count bound, i.e. a flush every 2^14 rows, what the kernel does for an index list that repeats rows.
  auto time_it = [&](Kind kind, int quant_bins, int n, int use_idx, RowBlockBound rb, int reps) -> float {
    HistWork hw = {0, n, use_idx, 0};
    CK(cudaMemcpy(d_work, &hw, sizeof(hw), cudaMemcpyHostToDevice));
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    float best = 1e30f, tot = 0;
    for (int r = 0; r < reps + 2; ++r) {
      CK(cudaMemsetAsync(d_hist, 0, slot_elems * 8));
      CK(cudaEventRecord(e0));
      const bool packed = kind == kPacked || kind == kPackedCount;
      if (use_idx) k_gather_q<<<nsm * 8, 256>>>(d_work, d_idx, d_idx, packed ? d_qp : d_q, d_qord);     // part of a leaf pass: timed
      launch(kind, quant_bins, d_qord, rb);
      CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
      if (r >= 2) { best = std::min(best, ms); tot += ms; }
    }
    (void)best;
    return tot / reps;
  };
  {  // one-time cost of the flush bound (a dataset computes it on first use): every bin byte read once, one shared atomic per byte
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0));
    launch_block_bound(d_bins, rows_stride, (int)N, num_tiles, F, d_bound, 0);
    CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    printf(" \"block_bound\": {\"ms\": %.3f, \"bin_bytes\": %zu},\n", ms, (size_t)num_tiles * N * 32);
  }
  printf(" \"k4_timing\": [\n");
  // packed rows (quantised training) at B = 4 and 16 beside <4> and <3>: their cap is 8191 and 2047 additions (a flush at least every
  // 7680 and 1536 rows of a bin-dense column).  The packed words are gen_q_packed's at B = 63; the timing does not depend on their values.
  struct Cfg { Kind kind; int quant_bins; double frac; int use_idx; int skew; int bound; };
  Cfg cfgs[] = {{kN4, 0, 1.0, 0, 0, 1}, {kN3, 0, 1.0, 0, 0, 1}, {kPacked, 4, 1.0, 0, 0, 1}, {kPacked, 16, 1.0, 0, 0, 1}, {kPackedCount, 4, 1.0, 0, 0, 1},
                {kN4, 0, 0.5, 1, 0, 1}, {kN4, 0, 0.1, 1, 0, 1}, {kPacked, 4, 0.1, 1, 0, 1}, {kN4, 0, 0.01, 1, 0, 1}, {kN4, 0, 0.001, 1, 0, 1},
                {kN4, 0, 1.0, 0, 1, 1}, {kN4, 0, 1.0, 0, 1, 0}, {kPacked, 4, 1.0, 0, 1, 1}};
  for (size_t c = 0; c < sizeof(cfgs) / sizeof(cfgs[0]); ++c) {
    int n = (int)(N * cfgs[c].frac);
    if (cfgs[c].use_idx) { gen_idx<<<nsm, 256>>>(d_idx, n, (int)(1.0 / cfgs[c].frac)); CK(cudaDeviceSynchronize()); }
    if (cfgs[c].skew && !cfgs[c - 1].skew) set_bins(0, (int)N);
    float ms = time_it(cfgs[c].kind, cfgs[c].quant_bins, n, cfgs[c].use_idx, cfgs[c].bound ? kb : RowBlockBound{nullptr, 0}, 5);
    double cells = (double)n * F;
    double bytes = (double)n * (F + 16.0 * num_tiles + (cfgs[c].use_idx ? 4.0 * num_tiles : 0.0)) + (double)F * 256 * 16;
    printf("  {\"kind\": \"%s\", \"quant_bins\": %d, \"rows\": %d, \"gather\": %d, \"skew\": %d, \"bound\": %d, \"ms\": %.4f, \"gcells_per_s\": %.2f, \"algo_GBps\": %.1f}%s\n",
           kind_name[cfgs[c].kind], cfgs[c].quant_bins, n, cfgs[c].use_idx, cfgs[c].skew, cfgs[c].bound, ms, cells / ms * 1e-6, bytes / ms * 1e-6,
           c + 1 < sizeof(cfgs) / sizeof(cfgs[0]) ? "," : "");
  }
  printf(" ]\n}\n");
  return (B200GBM_K4_EXPERIMENT == 0 && k4_bad != 0) ? 1 : 0;
}
