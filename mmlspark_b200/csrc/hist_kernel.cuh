// K4 — per-partition feature-histogram build (sm_90a).
//
// Replaces [UPSTREAM lightgbmlib 3.2.110] Dataset::ConstructHistograms /
// DenseBin<uint8>::ConstructHistogram, reached from the reference at
// lightgbm/src/main/scala/com/microsoft/ml/spark/lightgbm/booster/LightGBMBooster.scala:351-361
// (LGBM_BoosterUpdateOneIter).  SURVEY.md §8(a) row a4.
//
// Layout in HBM
//   bins : uint8 [num_tiles][rows_stride][32]   ("tile-major": a feature tile = 32 features,
//          one row of a tile = one 32-byte sector, so both the streamed root pass and the
//          index-list gather of a leaf move whole sectors)
//   qgh  : int4  [N]  per-row fixed-point gradient/hessian words {g_hi, g_lo, h_hi, h_lo}
//          (see quantize.h).  Written once per tree by the gradient kernel.
//   idx  : int32 row-index list of the data partition (leaves are contiguous ranges)
//   hist : int64 [num_feat_padded][256][2]  (g, h) fixed-point sums per leaf slot.
//
// Why fixed point: shared memory on sm_90a has exactly one native atomic add,
// ATOMS.ADD (32-bit integer).  atomicAdd on float/double/u64 in shared memory compiles to an
// ATOMS.CAST.SPIN compare-and-swap loop (checked with cuobjdump).  The reference accumulates
// fp32 gradients into fp64 bins, so fp32 accumulation is not good enough to reproduce its
// tree structure.  We therefore split a 36-bit fixed-point value into two 18-bit fields and
// accumulate each with a native 32-bit atomic; one (column, bin) cell can take 2^14 additions before a field can
// overflow, then the CTA flushes its sub-histogram into the int64 leaf histogram in L2 with TMA bulk
// reductions (UBLKRED.G.S.ADD.U64).  Integer sums are exact and order-independent, so the result is bit-reproducible
// run to run and across ranks (the NCCL reduction is an int64 sum).
//
// When to flush: a per-block bin-count bound of the dataset (k_block_maxcnt: for every tile and block of 4096 rows, the largest
// row count of any cell) bounds the additions a run of work items can put into one cell.  A CTA flushes when that bound would pass
// 2^14, when the tile changes, and after its last item.  Uniform 255-bin columns put ~16 rows per cell into a block, so a root-pass
// CTA flushes every few dozen 2^14-row items instead of after every one; a column with one dominant bin falls back to the latter.
//
// Bank mapping: the sub-histogram planes are laid out [bin][feature-of-tile], so feature f lives in
// bank f.  A consumer warp step is 32 rows x 4 features: lane = row for 8 steps, its (g,h) quadruple stays in registers
// (one 16-byte LDS per 32 cells), and the bin word and byte are rotated by the lane id, so every ATOMS instruction of a warp
// addresses 32 DIFFERENT features: conflict-free by construction regardless of the bin distribution (ncu: 1.0 wavefront per ATOMS).
// The LSU data pipe is the binding unit (ncu: ~94 % busy): an ATOMS wavefront costs ~0.93 cycles, so the loop spends
// 16 x 0.93 (atomics) + 1 (bin word) + 0.5 (q) cycles per 128 cells.  DESIGN.md §3 has the measurements and the rejected variants.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cuda_runtime.h>
#include <cub/block/block_scan.cuh>

namespace b200gbm {

constexpr int kTileFeat = 32;                      // features per tile == lanes per warp
constexpr int kBins = 256;                         // uint8 bin ids
constexpr int kLoBits = 18;                        // low fixed-point field
constexpr int kFlushRows = 1 << (32 - kLoBits);    // rows a sub-histogram may absorb (16384)
// Cost-model builds of k4_hist_build_ws for tools/ubench_hist.cu; every mode but 0 computes WRONG histograms.
//   1 / 2 / 3: the scatter loop issues 0 / 1 / 2 shared atomics per cell;
//   4: full scatter loop, the flush reads and zeroes the planes but sends nothing to the global histogram.
#ifndef B200GBM_K4_EXPERIMENT
#define B200GBM_K4_EXPERIMENT 0
#endif
constexpr int kPlaneWords = kBins * kTileFeat;     // 8192 words per plane

// Device-resident work descriptor: the controller kernels write it, so the host never has to
// know leaf sizes (no host sync inside a tree).
struct HistWork {
  int begin;      // first position in idx (or first row when use_idx == 0)
  int count;      // rows of the leaf on this rank
  int use_idx;    // 0: rows are begin..begin+count-1 directly (root of a full pass)
  int buf;        // which of the two index buffers holds the leaf's row list
};

// (g,h) words of a leaf in partition order: qord[begin + i] = qgh[idx[begin + i]] (no-op for the identity root)
__global__ void __launch_bounds__(256)
k_gather_q(const HistWork* __restrict__ work, const int* __restrict__ idx0, const int* __restrict__ idx1, const int4* __restrict__ qgh,
           int4* __restrict__ qord) {
  const HistWork w = *work;
  if (!w.use_idx) return;
  const int* __restrict__ idx = w.buf ? idx1 : idx0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < w.count; i += gridDim.x * blockDim.x) {
    const int p = w.begin + i;
    qord[p] = qgh[idx[p]];
  }
}

// ---------------------------------------------------------------------------------------------------
// Per-block bin-count bound of K4's flush rule.  The rows are cut into blocks of kBoundBlockRows; maxcnt(tile, block) is the largest
// number of the block's rows that fall into one (storage column, bin) cell of the tile.  It is kept as an exclusive prefix over the
// blocks of each tile, prefix[tile * (blocks + 1) + b] = sum of maxcnt over blocks < b, so any subset of the rows of blocks [b0, b1]
// adds at most prefix[b1 + 1] - prefix[b0] to one cell of the tile.  A tile's total is at most num_data <= 2^31 - 1: int does not
// overflow.  It depends on the bins only, so a dataset computes it once (Dataset::BlockBound).
constexpr int kBoundBlockRows = 4096;
struct RowBlockBound {
  const int* prefix;   // [num_tiles][blocks + 1]; nullptr: no bound, an item is bounded by its row count
  int blocks;
};
inline int bound_blocks(int num_data) { return (num_data + kBoundBlockRows - 1) / kBoundBlockRows; }

// grid (blocks, num_tiles): maxcnt of one (tile, block) into prefix[tile][block] (k_block_bound_prefix turns it into the prefix)
__global__ void __launch_bounds__(256)
k_block_maxcnt(const uint8_t* __restrict__ bins, size_t rows_stride, int num_data, int num_columns, int* __restrict__ prefix) {
  __shared__ unsigned cnt[kBins * kTileFeat];   // [bin][column of the tile]
  __shared__ unsigned wmax[8];
  const int tile = blockIdx.y, tid = threadIdx.x;
  for (int e = tid; e < kBins * kTileFeat; e += blockDim.x) cnt[e] = 0u;
  __syncthreads();
  const int r0 = blockIdx.x * kBoundBlockRows, rows = min(kBoundBlockRows, num_data - r0);
  const unsigned* wp = reinterpret_cast<const unsigned*>(bins + (static_cast<size_t>(tile) * rows_stride + r0) * kTileFeat);
  for (int e = tid; e < rows * 8; e += blockDim.x) {      // one 4-byte word = 4 columns of one row
    const unsigned word = wp[e];
    const int c0 = (e & 7) * 4, rot = (e >> 3) & 3;       // byte order rotated by the row: a warp's atomics hit 32 banks
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int kk = (k + rot) & 3;
      atomicAdd(&cnt[((word >> (8 * kk)) & 0xFFu) * kTileFeat + c0 + kk], 1u);
    }
  }
  __syncthreads();
  // Storage columns that no feature maps to (padding of the last tile) are left out: their bytes may put every row into one bin,
  // which would bound nothing.  No reader looks at their cells, and a 32-bit field that wraps there is defined behaviour.
  const int ncol = min(kTileFeat, num_columns - tile * kTileFeat);
  unsigned m = 0u;
  for (int e = tid; e < kBins * kTileFeat; e += blockDim.x)
    if ((e & (kTileFeat - 1)) < ncol) m = max(m, cnt[e]);
  m = __reduce_max_sync(0xffffffffu, m);
  if ((tid & 31) == 0) wmax[tid >> 5] = m;
  __syncthreads();
  if (tid == 0) {
    for (int i = 1; i < static_cast<int>(blockDim.x >> 5); ++i) m = max(m, wmax[i]);
    prefix[static_cast<size_t>(tile) * (gridDim.x + 1) + blockIdx.x] = static_cast<int>(m);
  }
}

// grid num_tiles: prefix[tile][0 .. blocks) holds maxcnt on entry; on exit prefix[tile][b] = sum of maxcnt over blocks < b, b = 0 .. blocks
__global__ void __launch_bounds__(1024) k_block_bound_prefix(int blocks, int* __restrict__ prefix) {
  using Scan = cub::BlockScan<int, 1024>;
  __shared__ typename Scan::TempStorage tmp;
  int* p = prefix + static_cast<size_t>(blockIdx.x) * (blocks + 1);
  int carry = 0;
  for (int b0 = 0; b0 < blocks; b0 += 1024) {
    const int b = b0 + threadIdx.x;
    const int v = b < blocks ? p[b] : 0;
    int ex, total;
    Scan(tmp).ExclusiveSum(v, ex, total);
    if (b < blocks) p[b] = carry + ex;
    carry += total;
    __syncthreads();      // tmp is reused by the next chunk
  }
  if (threadIdx.x == 0) p[blocks] = carry;
}

// prefix: [num_tiles][bound_blocks(num_data) + 1] ints
inline void launch_block_bound(const uint8_t* bins, size_t rows_stride, int num_data, int num_tiles, int num_columns, int* prefix,
                               cudaStream_t stream) {
  const int blocks = bound_blocks(num_data);
  if (blocks > 0) k_block_maxcnt<<<dim3(blocks, num_tiles), 256, 0, stream>>>(bins, rows_stride, num_data, num_columns, prefix);
  k_block_bound_prefix<<<num_tiles, 1024, 0, stream>>>(blocks, prefix);
}


__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem));
  int sz = valid ? 16 : 0;   // src-size 0 => zero fill, nothing is read
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(sz));
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

// ===================================================================================================
// k4_hist_build_ws is warp-specialised: two PRODUCER warps stage rows into a ring of shared-memory stages,
// 16 CONSUMER warps do nothing but the conflict-free scatter.  Stages are handed over with mbarriers
// (full / empty), so there is no block-wide barrier per stage and the producers run ahead across work
// items (they prefetch the next item while the consumers flush the current sub-histogram).
//   * contiguous row ranges (root pass, use_idx == 0): TMA bulk copies — one elected lane issues
//     cp.async.bulk (UBLKCP) for the stage's bins (rows*32 B) and qgh (rows*16 B), completion is signalled
//     by the mbarrier's transaction count;
//   * index-list leaves: all producer lanes issue 16-byte cp.async gathers (LDGSTS) and arrive on the
//     mbarrier with cp.async.mbarrier.arrive.noinc when their copies have landed.
constexpr int kWsConsumerWarps = 16;
constexpr int kWsProducerWarps = 2;                               // 1 lane issues the TMA bulk copies; all lanes share the gathers
constexpr int kWsThreads = (kWsConsumerWarps + kWsProducerWarps) * 32;
constexpr int kWsStageRows = 512;
constexpr int kWsStages = 3;
// Flush staging: one slab of 32 bins x 32 features as int64 (g,h) pairs laid out like the global histogram ([feature][bin][2]),
// one 512-byte row per feature.  Lane l handles feature l and slab bin (j + l) & 31 for j = warp and warp + 16: its plane word sits in bank l
// and the 8 lanes of a quarter-warp store their 16-byte pairs at 8 consecutive bin slots mod 8, so reads and stores are conflict-free
// without padding and every row stays 128-byte aligned for the bulk reduction.
constexpr int kFlushSlabBins = 32;
constexpr int kFlushRowBytes = kFlushSlabBins * 16;
constexpr int kFlushStageBytes = kTileFeat * kFlushRowBytes;     // 16 KB
constexpr int kWsSmemBytes = 4 * kPlaneWords * 4 + kWsStages * (kWsStageRows * 32 + kWsStageRows * 16) + kFlushStageBytes + 64;
static_assert(kWsSmemBytes <= 227 * 1024, "K4 shared memory exceeds the 227 KB per block of sm_90");
static_assert(kFlushSlabBins * kTileFeat == 2 * kWsConsumerWarps * 32, "a flush slab is two (g,h) pairs per consumer thread");

__device__ __forceinline__ unsigned smem_u32(const void* p) { return static_cast<unsigned>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* smem_dst, const void* gmem_src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(unsigned long long* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
// TMA bulk reduction: gmem[i] += smem[i] for bytes/8 u64 elements (UBLKRED.G.S.ADD.U64), tracked by the issuing thread's bulk groups.
// The PTX ISA (cp.reduce.async.bulk, ISA 8.0) gives each element's reduction .relaxed.gpu memory-ordering semantics, i.e. every
// element is an atomic read-modify-write at GPU scope, so the reductions of CTAs that flush the same feature tile concurrently all land.
__device__ __forceinline__ void bulk_reduce_add_u64(unsigned long long* gmem_dst, const void* smem_src, unsigned bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.u64 [%0], [%1], %2;\n" ::"l"(gmem_dst), "r"(smem_u32(smem_src)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;\n" ::: "memory"); }   // sources read
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;\n" ::: "memory"); }             // writes done
// generic-proxy shared-memory writes before this fence are visible to the async proxy (TMA) after the following barrier
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

// Quantised training (use_quantized_grad): the (g,h) words hold small integers, |q_g| <= floor(B/2) and |q_h| <= B (B =
// num_grad_quant_bins), or q_h = 1 on the count plane of constant hessians.  One packed plane then carries both: the lane builds
// w = (q_g << 16) + q_h once per row and a cell takes ONE 32-bit atomic (wrapping), instead of 4 (or 3).  As long as neither sum leaves
// [-32767, 32767], w's low 16 bits are the sign-extended h sum and (w - h) >> 16 the g sum.  A cell takes at most
// packed_flush_cap(B, count_plane) additions before a field could leave that range; it replaces kFlushRows in the flush rule.
inline int packed_flush_cap(int quant_bins, bool count_plane) {
  return 32767 / std::max(quant_bins / 2, count_plane ? 1 : quant_bins);
}

// The body of every K4 instantiation.  NATOM selects the planes: 4 = (g_hi,g_lo,h_hi,h_lo) general case, 3 = constant-hessian objectives
// (g_hi,g_lo,count) [UPSTREAM is_constant_hessian path], 1 = one packed plane of quantised training (above).  cap: the additions a
// cell may take between flushes (kFlushRows, or packed_flush_cap for NATOM 1, at least kWsStageRows); count_plane (NATOM 1 only):
// q_h is 1 per row instead of the words' h fields.
template <int NATOM>
__device__ __forceinline__ void k4_hist_body(const uint8_t* __restrict__ bins, size_t rows_stride, int num_tiles, const int4* __restrict__ qgh,
                                             const int4* __restrict__ qord, const int* __restrict__ idx0, const int* __restrict__ idx1,
                                             const HistWork* __restrict__ work, unsigned long long* __restrict__ hist, RowBlockBound bound,
                                             int cap, int count_plane) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  unsigned* plane = reinterpret_cast<unsigned*>(smem_raw);
  unsigned char* stage_bins = smem_raw + 4 * kPlaneWords * 4;
  int4* stage_q = reinterpret_cast<int4*>(stage_bins + kWsStages * kWsStageRows * 32);
  unsigned char* flush_stage = reinterpret_cast<unsigned char*>(stage_q) + kWsStages * kWsStageRows * 16;   // [feature][kFlushRowBytes]
  unsigned long long* full_bar = reinterpret_cast<unsigned long long*>(flush_stage + kFlushStageBytes);
  unsigned long long* empty_bar = full_bar + kWsStages;

  const HistWork w = *work;
  const int n = w.count;
  if (n <= 0) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int* __restrict__ idx = w.buf ? idx1 : idx0;

  // Work items are (tile, row chunk) pairs in TILE-MAJOR order; every CTA takes one contiguous range of them, so
  // consecutive items of a CTA mostly belong to the same feature tile and the sub-histogram is flushed only when the
  // tile changes or the bound of the items absorbed since the last flush could pass the cap of additions per cell (below).
  long long cells_rows = static_cast<long long>(n) * num_tiles;
  int rpi = static_cast<int>((cells_rows + 4LL * gridDim.x - 1) / (4LL * gridDim.x));
  rpi = (rpi + kWsStageRows - 1) / kWsStageRows * kWsStageRows;
  rpi = max(rpi, kWsStageRows);
  rpi = min(rpi, cap / kWsStageRows * kWsStageRows);
  const int chunks = (n + rpi - 1) / rpi;
  const long long items = static_cast<long long>(chunks) * num_tiles;
  const int i0 = static_cast<int>(items * blockIdx.x / gridDim.x);
  const int i1 = static_cast<int>(items * (blockIdx.x + 1) / gridDim.x);
  if (i0 >= i1) return;

  if (tid == 0) {
    for (int i = 0; i < kWsStages; ++i) { mbar_init(&full_bar[i], kWsProducerWarps * 32); mbar_init(&empty_bar[i], kWsConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  for (int e = tid; e < 4 * kPlaneWords; e += kWsThreads) plane[e] = 0u;
  __syncthreads();

  unsigned gs = 0;   // global stage counter (same sequence on both sides)
  if (warp >= kWsConsumerWarps) {
    // ------------------------------------------------------------------ producer warps
    const int ptid = tid - kWsConsumerWarps * 32;                 // 0 .. kWsProducerWarps*32-1
    constexpr int kPT = kWsProducerWarps * 32;
    constexpr int kPerLane = kWsStageRows / kPT;
    for (int item = i0; item < i1; ++item) {
      const int tile = item / chunks, chunk = item - tile * chunks;
      const int row0 = chunk * rpi;
      const int nrows = min(rpi, n - row0);
      const int nst = (nrows + kWsStageRows - 1) / kWsStageRows;
      const uint8_t* tbins = bins + static_cast<size_t>(tile) * rows_stride * 32;
      for (int s = 0; s < nst; ++s, ++gs) {
        const int slot = gs % kWsStages;
        mbar_wait(&empty_bar[slot], ((gs / kWsStages) & 1u) ^ 1u);
        const int p0 = row0 + s * kWsStageRows;
        const int rows = min(kWsStageRows, row0 + nrows - p0);
        unsigned char* db = stage_bins + slot * kWsStageRows * 32;
        int4* dq = stage_q + slot * kWsStageRows;
        if (!w.use_idx) {
          if (ptid == 0) {
            mbar_arrive_expect_tx(&full_bar[slot], static_cast<unsigned>(rows) * 48u);
            const size_t r = static_cast<size_t>(w.begin + p0);
            tma_bulk_g2s(db, tbins + r * 32, static_cast<unsigned>(rows) * 32u, &full_bar[slot]);
            tma_bulk_g2s(dq, qgh + r, static_cast<unsigned>(rows) * 16u, &full_bar[slot]);
          } else {
            mbar_arrive(&full_bar[slot]);
          }
        } else {
          // leaf = index list: the bin rows are gathered sector by sector with cp.async; the (g,h) words were put into LEAF ORDER
          // once per leaf by k_gather_q (qord[position]), so every feature tile streams them with one bulk copy instead of
          // re-gathering 16 B out of a 64 B DRAM atom 16 times (ncu: the per-tile q gather doubled the DRAM traffic of a leaf pass)
          const int* ip = idx + w.begin + p0;
          if (ptid == 0) {
            mbar_expect_tx(&full_bar[slot], static_cast<unsigned>(rows) * 16u);
            tma_bulk_g2s(dq, qord + static_cast<size_t>(w.begin + p0), static_cast<unsigned>(rows) * 16u, &full_bar[slot]);
          }
          // (one 32-byte cp.async.bulk per row was tried instead: the TMA unit retires ~1 such copy per 32 cycles per SM, 4.5x slower)
          // a lane pair fetches the two 16-byte halves of ONE row sector, so an LDGSTS instruction touches 16 sectors instead of
          // 32 (ncu: the data return costs one LSU wavefront per distinct sector: 28 per instruction with one half-row per lane)
          int rr[2 * kPerLane];
#pragma unroll
          for (int k = 0; k < 2 * kPerLane; ++k) { const int j = (ptid + k * kPT) >> 1; rr[k] = j < rows ? ip[j] : -1; }
#pragma unroll
          for (int k = 0; k < 2 * kPerLane; ++k) {
            const int hh = ptid + k * kPT, j = hh >> 1, half = (hh & 1) * 16;
            if (rr[k] >= 0) cp_async16(db + j * 32 + half, tbins + static_cast<size_t>(rr[k]) * 32 + half, true);
          }
          cp_async_mbar_arrive_noinc(&full_bar[slot]);
        }
      }
    }
    cp_async_wait<0>();
  } else {
    // ------------------------------------------------------------------ consumer warps
    // Warp step = 32 rows x 4 features: lane owns ROW g*32+lane for 8 steps and keeps its (g,h) quadruple in registers, so the
    // 16-byte q load (4 LSU wavefronts for a warp) is paid once per 1024 cells instead of once per 128.  At step k the lane reads
    // bin word w = ((lane>>2)+k)&7 of its row: bank = 8*(lane&3)+w, all 32 distinct.  Inside the word the byte order is rotated
    // by lane&3, so the 32 atomics of one instruction hit features 4w+kk = 32 distinct banks (plane index = bin*32 + feature).
#if B200GBM_K4_EXPERIMENT >= 1 && B200GBM_K4_EXPERIMENT <= 3
    unsigned exp_sink = 0;
#endif
    const int sub = lane >> 2, rot = lane & 3;
    // Most additions one cell of the item's tile can take from the item: its row count, or the block bound of the rows between its
    // first and last row.  Index-list items take those two rows from the list: every leaf's row list is strictly ascending (the
    // identity root, k_bag_compact's in-bag list and the stable k_partition scatter all keep the row order), so all rows of the
    // item lie in between.  Every consumer thread reads the same values and so reaches the same flush decision.
    // The loads run two items ahead, so no consumer waits on them: the first and last row of item k + 2 and the bound of item
    // k + 1 are loaded when item k starts, and that bound is first used when item k ends.
    auto item_rows = [&](int it, int& first, int& last) {
      const int t = it / chunks, r0 = (it - t * chunks) * rpi;
      first = w.begin + r0;
      last = first + min(rpi, n - r0) - 1;
      if (w.use_idx && bound.prefix) { first = idx[first]; last = idx[last]; }
    };
    auto item_bound = [&](int it, int first, int last) -> int {
      const int t = it / chunks, nr = min(rpi, n - (it - t * chunks) * rpi);
      if (!bound.prefix) return nr;
      const int* p = bound.prefix + static_cast<size_t>(t) * (bound.blocks + 1);
      return min(nr, p[last / kBoundBlockRows + 1] - p[first / kBoundBlockRows]);
    };
    int first, last;                                              // first and last row of the item whose bound is loaded next
    item_rows(i0, first, last);
    int next_bound = item_bound(i0, first, last);
    if (i0 + 1 < i1) item_rows(i0 + 1, first, last);
    int acc_bound = 0;                                            // bound of the items absorbed since the last flush, <= kFlushRows
    for (int item = i0; item < i1; ++item) {
      const int tile = item / chunks, chunk = item - tile * chunks;
      const int row0 = chunk * rpi;
      const int nrows = min(rpi, n - row0);
      const int nst = (nrows + kWsStageRows - 1) / kWsStageRows;
      acc_bound += next_bound;
      next_bound = 0;
      if (item + 1 < i1) {
        next_bound = item_bound(item + 1, first, last);
        if (item + 2 < i1) item_rows(item + 2, first, last);
      }
      for (int s = 0; s < nst; ++s, ++gs) {
        const int slot = gs % kWsStages;
        mbar_wait(&full_bar[slot], (gs / kWsStages) & 1u);
        const int rows = min(kWsStageRows, nrows - s * kWsStageRows);
        const unsigned* sw = reinterpret_cast<const unsigned*>(stage_bins + slot * kWsStageRows * 32);
        const int4* sq = stage_q + slot * kWsStageRows;
        const int groups = (rows + 31) >> 5;
        for (int g = warp; g < groups; g += kWsConsumerWarps) {
          const int r = g * 32 + lane;
          if (r < rows) {
            const int4 q = sq[r];
            unsigned packed = 0u;
            if (NATOM == 1) {
              const int qg = (q.x << kLoBits) + q.y, qh = count_plane ? 1 : (q.z << kLoBits) + q.w;
              packed = (static_cast<unsigned>(qg) << 16) + static_cast<unsigned>(qh);
            }
            const unsigned* rw = sw + r * 8;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              const int w8 = (sub + k) & 7;
              const unsigned word = rw[w8];
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const int kk = (j + rot) & 3;
                const unsigned b = (word >> (8 * kk)) & 0xFFu;
                const unsigned a = b * 32u + static_cast<unsigned>(w8 * 4 + kk);
#if B200GBM_K4_EXPERIMENT == 0 || B200GBM_K4_EXPERIMENT == 4
                if (NATOM == 1) {
                  atomicAdd(&plane[a], packed);
                } else {
                  atomicAdd(&plane[a], static_cast<unsigned>(q.x));
                  atomicAdd(&plane[kPlaneWords + a], static_cast<unsigned>(q.y));
                  atomicAdd(&plane[2 * kPlaneWords + a], static_cast<unsigned>(q.z));
                  if (NATOM == 4) atomicAdd(&plane[3 * kPlaneWords + a], static_cast<unsigned>(q.w));
                }
#else   // tools/ubench_hist.cu only: cost model of the loop with 0 / 1 / 2 atomics per cell
                if (B200GBM_K4_EXPERIMENT >= 2) atomicAdd(&plane[a], static_cast<unsigned>(q.x));
                if (B200GBM_K4_EXPERIMENT >= 3) atomicAdd(&plane[kPlaneWords + a], static_cast<unsigned>(q.y));
                if (B200GBM_K4_EXPERIMENT == 1) exp_sink ^= a + static_cast<unsigned>(q.x ^ q.y ^ q.z ^ q.w);
                (void)packed;
#endif
              }
            }
          }
        }
#if B200GBM_K4_EXPERIMENT >= 1 && B200GBM_K4_EXPERIMENT <= 3
        if (exp_sink == 0x12345679u) plane[lane] = exp_sink;
#endif
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[slot]);
      }
      // rpi <= cap, so a single item never breaks the bound
      const bool flush = (item + 1 == i1) || ((item + 1) / chunks != tile) || (acc_bound + next_bound > cap);
      if (!flush) continue;
      acc_bound = 0;
      // All consumers finished: flush the sub-histogram into the int64 leaf histogram (consumer-only named barriers; the producers
      // keep staging).  Slab by slab (32 bins x 32 features), every consumer thread reads and re-zeroes the plane words of two
      // (bin, feature) cells, combines them into int64 (g,h) and stores the pairs into the staging buffer in the histogram's own
      // [feature][bin][2] order; thread 0 then sends each feature's 512-byte run to L2 with one TMA bulk reduction.  Scattered
      // 64-bit REDs (one cache line per lane, all through the LSU) cost 19-40 % of the kernel's time on H100 (DESIGN.md §3); the bulk
      // reductions run in the TMA unit beside the next slab's plane reads and the next item's atomics.
      asm volatile("bar.sync 1, %0;\n" ::"n"(kWsConsumerWarps * 32) : "memory");
      unsigned long long* htile = hist + static_cast<size_t>(tile) * kTileFeat * kBins * 2;
      int sbin[2];                                                  // slab bin of this thread's two cells; its feature is `lane`
#pragma unroll
      for (int i = 0; i < 2; ++i) sbin[i] = (warp + i * kWsConsumerWarps + lane) & (kFlushSlabBins - 1);
      for (int b0 = 0; b0 < kBins; b0 += kFlushSlabBins) {
        long long g[2], h[2];
        bool nz = false;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int e = (b0 + sbin[i]) * kTileFeat + lane;          // plane index = bin*32 + feature
          if (NATOM == 1) {
            const unsigned pw = plane[e];
            plane[e] = 0u;
            nz |= pw != 0u;
            const int ph = static_cast<int>(static_cast<short>(pw & 0xFFFFu));      // sext16 of the low field
            g[i] = (static_cast<int>(pw) - ph) >> 16;
            h[i] = ph;
            continue;
          }
          const unsigned ghi = plane[e], glo = plane[kPlaneWords + e], hhi = plane[2 * kPlaneWords + e];
          const unsigned hlo = (NATOM == 4) ? plane[3 * kPlaneWords + e] : 0u;
          plane[e] = 0u;
          plane[kPlaneWords + e] = 0u;
          plane[2 * kPlaneWords + e] = 0u;
          if (NATOM == 4) plane[3 * kPlaneWords + e] = 0u;
          nz |= (ghi | glo | hhi | hlo) != 0u;
          g[i] = (static_cast<long long>(static_cast<int>(ghi)) << kLoBits) + static_cast<long long>(glo);
          h[i] = (NATOM == 4) ? (static_cast<long long>(static_cast<int>(hhi)) << kLoBits) + static_cast<long long>(hlo)
                              : static_cast<long long>(hhi);   // plain row count
        }
        // the previous slab's reductions must have read the staging buffer before it is overwritten
        if (tid == 0) bulk_wait_read_all();
        asm volatile("bar.sync 1, %0;\n" ::"n"(kWsConsumerWarps * 32) : "memory");
#pragma unroll
        for (int i = 0; i < 2; ++i)
          *reinterpret_cast<longlong2*>(flush_stage + lane * kFlushRowBytes + sbin[i] * 16) = make_longlong2(g[i], h[i]);
        fence_proxy_async_smem();
        // barrier + OR of "this slab has a non-zero cell": an all-zero slab (small leaves) sends nothing
        int any;
        asm volatile(
            "{\n"
            ".reg .pred p, q;\n"
            "setp.ne.u32 p, %1, 0;\n"
            "bar.red.or.pred q, 1, %2, p;\n"
            "selp.s32 %0, 1, 0, q;\n"
            "}\n"
            : "=r"(any)
            : "r"(static_cast<unsigned>(nz)), "n"(kWsConsumerWarps * 32)
            : "memory");
#if B200GBM_K4_EXPERIMENT != 4
        if (tid == 0 && any) {
          for (int f = 0; f < kTileFeat; ++f)
            bulk_reduce_add_u64(htile + (static_cast<size_t>(f) * kBins + b0) * 2, flush_stage + f * kFlushRowBytes, kFlushSlabBins * 16);
          bulk_commit();
        }
#else
        (void)any; (void)htile;
#endif
      }
      // the planes are zero again (every plane write precedes the last barrier above); the staging buffer is guarded by the wait
    }
    // the bulk reductions read shared memory and write the histogram that the next kernel scans: complete them before exiting
    if (tid == 0) bulk_wait_all();
  }
}

// The full-precision instantiations <4> and <3>: their cap is the compile-time kFlushRows.
template <int NATOM>
__global__ void __launch_bounds__(kWsThreads, 1)
k4_hist_build_ws(const uint8_t* __restrict__ bins, size_t rows_stride, int num_tiles, const int4* __restrict__ qgh,
                 const int4* __restrict__ qord, const int* __restrict__ idx0, const int* __restrict__ idx1,
                 const HistWork* __restrict__ work, unsigned long long* __restrict__ hist, RowBlockBound bound) {
  k4_hist_body<NATOM>(bins, rows_stride, num_tiles, qgh, qord, idx0, idx1, work, hist, bound, kFlushRows, 0);
}

// The packed instantiation of quantised training: cap = packed_flush_cap(B, count_plane), >= kWsStageRows for B <= 63.
__global__ void __launch_bounds__(kWsThreads, 1)
k4_hist_build_packed(const uint8_t* __restrict__ bins, size_t rows_stride, int num_tiles, const int4* __restrict__ qgh,
                     const int4* __restrict__ qord, const int* __restrict__ idx0, const int* __restrict__ idx1,
                     const HistWork* __restrict__ work, unsigned long long* __restrict__ hist, RowBlockBound bound, int cap, int count_plane) {
  k4_hist_body<1>(bins, rows_stride, num_tiles, qgh, qord, idx0, idx1, work, hist, bound, cap, count_plane);
}

// K4's shared memory exceeds the 48 KB default: raise the limit of every instantiation on the current device.  Call it once per
// device at set-up; it is host work that does not belong in the per-split launches.
inline cudaError_t set_k4_smem_limit() {
  cudaError_t e = cudaFuncSetAttribute(k4_hist_build_ws<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, kWsSmemBytes);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(k4_hist_build_ws<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kWsSmemBytes);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(k4_hist_build_packed, cudaFuncAttributeMaxDynamicSharedMemorySize, kWsSmemBytes);
}

// One persistent K4 launch: `grid` is one CTA per SM; constant-hessian objectives accumulate 3 planes (g_hi, g_lo, count).
// quant_bins > 0 (quantised training, the words hold K3's discretised q): the packed plane with that B's cap, q_h = 1 per row when
// const_hessian.  `bound` is the bins' per-block bound (launch_block_bound); index lists given with it must be strictly ascending.
inline void launch_k4(bool const_hessian, int quant_bins, const uint8_t* bins, size_t rows_stride, int num_tiles, const int4* qgh,
                      const int4* qord, const int* idx0, const int* idx1, const HistWork* work, unsigned long long* hist, RowBlockBound bound,
                      int grid, cudaStream_t stream) {
  if (quant_bins > 0)
    k4_hist_build_packed<<<grid, kWsThreads, kWsSmemBytes, stream>>>(bins, rows_stride, num_tiles, qgh, qord, idx0, idx1, work, hist, bound,
                                                                    packed_flush_cap(quant_bins, const_hessian), const_hessian ? 1 : 0);
  else if (const_hessian)
    k4_hist_build_ws<3><<<grid, kWsThreads, kWsSmemBytes, stream>>>(bins, rows_stride, num_tiles, qgh, qord, idx0, idx1, work, hist, bound);
  else
    k4_hist_build_ws<4><<<grid, kWsThreads, kWsSmemBytes, stream>>>(bins, rows_stride, num_tiles, qgh, qord, idx0, idx1, work, hist, bound);
}

}  // namespace b200gbm
