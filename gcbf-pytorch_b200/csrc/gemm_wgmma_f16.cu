// wgmma GEMM with error-compensated 3xFP16 arithmetic -- the fast path of the linear layers of gcbf.nn.MLP
// (reference gcbf/nn/mlp.py:44-47; the 2048-wide phi / gamma GEMMs are > 99 % of the FLOPs of a GCBF.update step).
//
// Precision.  The parity bar (h, u, loss within 1e-5 of the fp32 reference) rules out plain TF32 / bf16 / fp16 operands.
// Every fp32 operand x is scaled by a per-tensor power of two s (max|x|*s in [2^14, 2^15), exact) and split
//        x*s = hi + lo,   hi = fp16(x*s),   lo = fp16(x*s - hi)            (22 significand bits together)
// and a product is accumulated in fp32 registers as  hi*hi + lo*hi + hi*lo  (3 wgmma f16 per k-slice; lo*lo ~ 2^-22
// is dropped) and descaled by 1/(s_a*s_b) when a chunk is promoted.  Same 22-bit operand precision as a 3xTF32 scheme at
// twice the tensor-core rate (an f16 wgmma consumes 16 K-elements per instruction, a tf32 one 8).  Elements more than 2^17 below the
// tensor's max lose relative (not absolute) precision: their absolute error stays <= 2^-39 of the max.
//
// "Split once, use everywhere".  The [hi | lo] fp16 companion of a matrix has the *same row-major layout* as the matrix,
// and the tensor core takes either operand K-major or MN-major, so one companion serves every GEMM the matrix is in:
//        forward      Y  = X  * W^T     A = X  (K-major)     B = W  (K-major)
//        data-grad    dX = dZ * W       A = dZ (K-major)     B = W  (MN-major)
//        weight-grad  dW = dZ^T * X     A = dZ (MN-major)    B = X  (MN-major)
// No transposes, no padding copies: TMA zero-fills ragged edges of the exact-size tensor maps.
//
// Kernel.  One CTA per 128 x BN output tile (BN = 128 or 256) and contraction split, three warpgroups: warp 0 of warpgroup 0
// is the TMA producer (cp.async.bulk.tensor 2-D boxes into swizzled shared memory, STAGES-deep mbarrier ring), warpgroups
// 1 and 2 each own 64 rows of the tile and issue m64n128k16 wgmma.  The producer warpgroup lowers its register budget to 40
// per thread and the consumer warpgroups raise theirs to 232 (setmaxnreg).  A 256-wide tile is computed as two 128-wide halves
// one after the other: the promoted sums of a half are parked in shared memory (the first half in its own buffer, the second
// in the drained stage ring), so every consumer thread holds 2 x 64 chunk + 64 promoted accumulators.  The tensor core's fp32
// accumulation truncates, so K is consumed in chunks of KCH k-blocks: each chunk starts from zero in the wgmma accumulators
// and is added to the promoted sums with one round-to-nearest FMA (which also applies the chunk's descale factor).  The
// tensor pipe is not drained between k-blocks: one k-block stays in flight (wait_group 1, its stage is released when the next
// one is committed), and consecutive chunks -- across the half boundary too -- alternate between two accumulator sets, so a
// chunk is promoted (and the first half parked) while the next chunk's MMAs run.  Summation order and roundings are those of
// a synchronous loop, so results do not depend on the schedule.  The epilogue then works on the whole parked tile: bias,
// activation / ReLU mask, tile maximum, fp32 output, fp16 companion, column sums.
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>

#include <atomic>

#include "common.cuh"
#include "sm90_ptx.cuh"

namespace gcbf {
namespace th {

using namespace ptx;

constexpr int BM = 128;
constexpr int BK = 32;                 // K elements per k-block (= one smem stage): 64-byte K-major rows
constexpr int SUB_N = 128;             // output columns per wgmma pass (m64n128k16)
constexpr int WG_K = 16;               // fp16: 32 bytes of K per instruction
constexpr int NUM_THREADS = 384;       // warpgroup 0: TMA producer (one thread); warpgroups 1-2: MMA + epilogue
constexpr int EPI_THREADS = 256;
constexpr int KCH_MAX = 256 / BK;      // k-blocks accumulated inside the tensor core before promotion to registers: upper limit (256 K-elements)
constexpr int MN_BOX = 64;             // MN-major operands: one TMA box = 64 MN elements (128 B, SWIZZLE_128B) x BK k-rows
constexpr int A_BYTES = BM * BK * 2;                         // one of hi / lo
constexpr int B_BYTES = SUB_N * BK * 2;
constexpr int RING_BYTES = 128 * 1024;                       // the stage ring, the same size for both product counts
// Products per k-slice P: 3 = hi*hi + lo*hi + hi*lo (fp32-grade, the default), 1 = hi*hi only (fp16 operands).  A P = 1 stage holds
// only the hi planes (16 KB), so the same ring is 8 stages deep instead of 4: a k-block has a third of the MMAs of a P = 3 one and
// half its bytes, and the deeper ring keeps twice as many k-blocks of loads in flight to feed it.
template <int P> __host__ __device__ constexpr int stage_bytes() { return P == 3 ? 2 * A_BYTES + 2 * B_BYTES : A_BYTES + B_BYTES; }   // 32 / 16 KB
template <int P> __host__ __device__ constexpr int stages() { return RING_BYTES / stage_bytes<P>(); }                                // 4 / 8
constexpr int PARK_PITCH = SUB_N + 8;                        // floats; conflict-free float2 stores of the accumulator fragments
constexpr int PARK_BYTES = BM * PARK_PITCH * 4;
static_assert(PARK_BYTES <= RING_BYTES, "the second half of a 256-wide tile is parked in the stage ring");
static_assert(2 * stages<1>() * 8 + (256 / 32) * 4 <= 256, "barriers and reduction words fit their 256 bytes");
constexpr int SMEM_BYTES = RING_BYTES + PARK_BYTES + 1024 /*align slack*/ + 256 /*barriers, reductions*/;

enum { EPI_FWD = 0, EPI_DGRAD = 1, EPI_WGRAD = 2 };

struct EpiParams {
  int mode;
  const float* alpha;          // device scalar (1/sigma of the spectral norm) or null
  const float* bias;
  int act;
  const float* relu_src;       // data-grad: ReLU mask source as fp32 (mask = src > 0) ...
  int ld_relu;
  const __half* relu_hi;       // ... or as the hi plane of the layer output's companion (mask = hi > 0)
  int ld_relu_h;
  int accumulate;
  size_t split_stride;         // split-K: contraction split blockIdx.y writes its own slice C + blockIdx.y * split_stride
  // amax words of the operands' companions: one per tensor (strides 0) or one per (128-row, 256-column) tile of the operand's own
  // matrix (strides in words: *_sr per row block, *_sc per column tile)
  const uint32_t* amax_a; int a_sr, a_sc;
  const uint32_t* amax_b; int b_sr, b_sc;
  uint32_t* amax_out;          // optional: atomicMax of |output| (feeds the next layer's split), or null
  // tile-scaled fp16 [hi|lo] companion of the OUTPUT, written by the epilogue (BN == 256 only): every CTA knows the exact max of its
  // 128 x 256 tile, so the scale needs neither a pass over the tensor nor an a-priori bound
  __half* out_h;               // hi plane; the lo plane follows at out_h + Mo * ld_out_h
  int ld_out_h;
  uint32_t* out_tile_amax;     // [ceil(Mo/128)][out_amax_stride] float bits of the tile maxima
  int out_amax_stride;
  float* colsum;               // optional: column sums of the (masked) output, one row of partials per row tile ([tiles_m][No])
};

// power-of-two scale s with amax*s in [2^14, 2^15); 1 for zero / denormal / non-finite amax
__host__ __device__ __forceinline__ uint32_t scale_bits_from_amax(uint32_t amax_bits) {
  const int e = (int)((amax_bits >> 23) & 0xffu);
  if (e == 0 || e == 255) return 0x3f800000u;
  int se = 127 + 14 - (e - 127);
  se = se < 2 ? 2 : (se > 252 ? 252 : se);
  return (uint32_t)se << 23;
}
__host__ __device__ __forceinline__ uint32_t inv_pow2_bits(uint32_t s_bits) { return (uint32_t)(254 - (int)(s_bits >> 23)) << 23; }

// descriptor of the k-slice `kk` (16 K-elements) of an operand tile in shared memory
template <bool MN_MAJOR>
__device__ __forceinline__ uint64_t tile_desc(uint32_t tile_addr, int kk) {
  if (MN_MAJOR) {
    // [MN/64 boxes][BK k-rows][64 MN elements]: 8 k-rows x 128 B = one swizzle atom; k-groups 1024 B apart (SBO),
    // 64-wide MN atoms BK*128 B apart (LBO)
    return make_smem_desc(tile_addr + (uint32_t)(kk * WG_K * 128), BK * 128, 1024, 128);
  }
  // [rows][BK k-elements] = 64-byte rows, SWIZZLE_64B: 8-row atoms 512 B apart (SBO); +32 B per k-slice inside the row
  return make_smem_desc(tile_addr + (uint32_t)(kk * WG_K * 2), 16, 8 * BK * 2, BK * 2);
}

template <bool MN_MAJOR>
__device__ __forceinline__ void load_tile(uint8_t* dst, const CUtensorMap* map, uint64_t* bar, int mn0, int k0, int rows) {
  if (MN_MAJOR) {
    for (int j = 0; j < rows / MN_BOX; ++j) tma_load_2d(dst + j * (BK * 128), map, bar, mn0 + j * MN_BOX, k0);
  } else {
    tma_load_2d(dst, map, bar, k0, mn0);
  }
}

__device__ __forceinline__ void epi_sync() { asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory"); }

// grid (tiles_m * tiles_n, contraction splits).  P = 1: the lo maps are not read (the launcher passes the hi maps in their place).
template <int BN, bool A_MN, bool B_MN, int P>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_h_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
              const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo,
              float* __restrict__ C, int ldc, int Mo, int No, int tiles_n, int kblocks_per_split, int kblocks_total, int KCH, EpiParams ep) {
  static_assert(P == 3 || P == 1, "products per k-slice: 3 (3xFP16) or 1 (fp16)");
  constexpr int STAGES = stages<P>();
  constexpr int STAGE_BYTES = stage_bytes<P>();
  constexpr int B_OFF = (P == 3 ? 2 : 1) * A_BYTES;       // stage layout: [A hi][A lo][B hi][B lo], or [A hi][B hi]
  constexpr int NSUB = BN / SUB_N;
  constexpr int MODE = A_MN ? EPI_WGRAD : (B_MN ? EPI_DGRAD : EPI_FWD);   // the operand layouts identify the product
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* park0 = reinterpret_cast<float*>(smem + RING_BYTES);            // columns [0, 128) of the tile
  float* park1 = reinterpret_cast<float*>(smem);                          // columns [128, 256): the drained stage ring
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + RING_BYTES + PARK_BYTES);
  uint64_t* full = bars;                        // [STAGES]  TMA -> MMA
  uint64_t* empty = bars + STAGES;              // [STAGES]  MMA -> TMA (one arrive per consumer warpgroup)
  uint32_t* red = reinterpret_cast<uint32_t*>(bars + 2 * STAGES);   // [EPI_THREADS / 32] per-warp maxima

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kb0 = blockIdx.y * kblocks_per_split;
  const int kb1 = min(kblocks_total, kb0 + kblocks_per_split);
  const int nkb = kb1 - kb0;
  const int m0 = (blockIdx.x / tiles_n) * BM, n0t = (blockIdx.x % tiles_n) * BN;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a_hi);
    if (P == 3) tma_prefetch_desc(&map_a_lo);
    tma_prefetch_desc(&map_b_hi);
    if (P == 3) tma_prefetch_desc(&map_b_lo);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  // 384 threads x 168 registers are allocated at launch; the producer warpgroup gives 128 back per thread, the two consumer
  // warpgroups take 64 more each: two chunk accumulator sets and the promoted sums fit (128 x 40 + 256 x 232 <= 64 K)
  if (warp < 4) {
    setmaxnreg_dec<40>();
    // ===== TMA producer =====
    if (threadIdx.x == 0) {
      // data-grad: once the first ring of loads is out, the tile's ReLU mask rows are requested into L2, so the epilogue does not
      // wait on HBM for them.  Whole 16-byte pieces inside the tile's columns only (a ragged tail is left to the epilogue's loads).
      bool mask_pending = MODE == EPI_DGRAD && (ep.relu_hi || ep.relu_src);
      auto prefetch_mask = [&]() {
        const int cols = min(BN, No - n0t), rows = min(BM, Mo - m0);
        const bool vec = !ep.relu_src || ((ep.ld_relu & 3) == 0 && (reinterpret_cast<uintptr_t>(ep.relu_src) & 15) == 0);
        const uint32_t bytes = (uint32_t)(cols * (ep.relu_src ? 4 : 2)) & ~15u;
        if (vec && bytes)
          for (int r = 0; r < rows; ++r)
            bulk_prefetch_l2(ep.relu_src ? static_cast<const void*>(ep.relu_src + (size_t)(m0 + r) * ep.ld_relu + n0t)
                                         : static_cast<const void*>(ep.relu_hi + (size_t)(m0 + r) * ep.ld_relu_h + n0t), bytes);
      };
      int stage = 0;
      uint32_t phase = 0;
      for (int sub = 0; sub < NSUB; ++sub) {
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* st = smem + stage * STAGE_BYTES;
          mbar_expect_tx(&full[stage], STAGE_BYTES);
          load_tile<A_MN>(st, &map_a_hi, &full[stage], m0, kb * BK, BM);
          if (P == 3) load_tile<A_MN>(st + A_BYTES, &map_a_lo, &full[stage], m0, kb * BK, BM);
          load_tile<B_MN>(st + B_OFF, &map_b_hi, &full[stage], n0t + sub * SUB_N, kb * BK, SUB_N);
          if (P == 3) load_tile<B_MN>(st + B_OFF + B_BYTES, &map_b_lo, &full[stage], n0t + sub * SUB_N, kb * BK, SUB_N);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
          if (mask_pending && (stage == 0 || kb + 1 == kb1)) { prefetch_mask(); mask_pending = false; }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    if (nkb > 0) {
      // ===== consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64) =====
      const int tid = threadIdx.x - 128;
      const int wg = tid >> 7;
      const int wl = (tid >> 5) & 3;            // warp inside the warpgroup: fragment rows 16 wl .. 16 wl + 15
      const bool leader = (tid & 127) == 0;     // arrives on empty[] for the warpgroup
      // A sub-tile of this warpgroup: K-major 64 rows x 64 B = 4096 B in; MN-major the second 64-wide box, also 4096 B in
      const uint32_t a_off = (uint32_t)wg * 4096u;
      // The chunks of both halves form one sequence g = sub * nch + c, accumulated alternately in d0 / d1 (chunk g in d[g & 1]).
      // One k-block stays in flight: after committing a k-block the warpgroup waits for the one before it, releases that one's
      // stage, and -- when the new k-block opened a chunk -- promotes the previous chunk from the other buffer (parking the first
      // half after its last chunk) while the tensor core works on the new one.  Chunk sums, promotion order and roundings are
      // those of a fully synchronous loop; only the waits move.
      const int nch = (nkb + KCH - 1) / KCH;    // promotion chunks per 128-column half
      // the chunk count through an empty asm: when the compiler can see that it is even (NSUB = 2) it drops the exit after d0,
      // and ptxas then serialises every wgmma of the loop (C7514)
      int nchunks = NSUB * nch;
      asm("" : "+r"(nchunks));
      int stage = 0;                            // stage / parity of the next k-block
      uint32_t phase = 0;
      int held = -1;                            // stage of the k-block in flight (released after the next one is committed)
      float cs_prev = 0.f;                      // descale of the chunk awaiting promotion
      float acc[64], d0[64], d1[64];
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] = 0.f;

      // park the promoted sums: fragment element j of lane l in warp wl is (row 16 wl + l/4 + 8 ((j/2)&1), column 8 (j/4) + 2 (l%4) + j%2)
      auto park_acc = [&](float* park) {
        const int r0 = wg * 64 + wl * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < 64; j += 4) {
          const int c = 8 * (j >> 2) + 2 * (lane & 3);
          *reinterpret_cast<float2*>(park + r0 * PARK_PITCH + c) = make_float2(acc[j], acc[j + 1]);
          *reinterpret_cast<float2*>(park + (r0 + 8) * PARK_PITCH + c) = make_float2(acc[j + 2], acc[j + 3]);
        }
      };
      // add a finished chunk sum into the promoted accumulators (one round-to-nearest fp32 FMA each)
      auto promote = [&](float (&p)[64], float cs) {
#pragma unroll
        for (int j = 0; j < 64; ++j) fence_operand(p[j]);
#pragma unroll
        for (int j = 0; j < 64; ++j) acc[j] = __fmaf_rn(p[j], cs, acc[j]);
      };
      // chunk g into d (its first wgmma overwrites d: scale_d = 0); p holds chunk g - 1 (still in flight when g > 0)
      auto run_chunk = [&](float (&d)[64], float (&p)[64], int g) {
        const int sub = (NSUB > 1 && g >= nch) ? 1 : 0;
        const int kc = (g - sub * nch) * KCH;
        // descale factor of this chunk: 1 / (s_a * s_b), powers of two.  Per-tensor companions: the same word every chunk;
        // tile-scaled companions: the word of the (128-row, 256-column) tile of the operand this chunk's k-range lies in.
        // Read here, a chunk before the promotion that uses it.
        const int n0 = n0t + sub * SUB_N;
        const int kstart = (kb0 + kc) * BK;
        const int ia = A_MN ? (kstart >> 7) * ep.a_sr + (m0 >> 8) * ep.a_sc : (m0 >> 7) * ep.a_sr + (kstart >> 8) * ep.a_sc;
        const int ib = B_MN ? (kstart >> 7) * ep.b_sr + (n0 >> 8) * ep.b_sc : 0;
        const float cs = __uint_as_float(inv_pow2_bits(scale_bits_from_amax(__ldg(ep.amax_a + ia)))) *
                         __uint_as_float(inv_pow2_bits(scale_bits_from_amax(__ldg(ep.amax_b + ib))));
        const int kend = min(nkb, kc + KCH);
        for (int kb = kc; kb < kend; ++kb) {
          mbar_wait(&full[stage], phase);
          const uint32_t st = smem_u32(smem + stage * STAGE_BYTES);
          const uint32_t a_hi = st + a_off, a_lo = st + A_BYTES + a_off, b_hi = st + B_OFF, b_lo = st + B_OFF + B_BYTES;
#pragma unroll
          for (int j = 0; j < 64; ++j) fence_operand(d[j]);
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < BK / WG_K; ++kk) {
            if constexpr (P == 3) {
              const uint64_t dah = tile_desc<A_MN>(a_hi, kk), dal = tile_desc<A_MN>(a_lo, kk);
              const uint64_t dbh = tile_desc<B_MN>(b_hi, kk), dbl = tile_desc<B_MN>(b_lo, kk);
              wgmma_m64n128k16_f16<A_MN ? 1 : 0, B_MN ? 1 : 0>(d, dal, dbh, (kb > kc || kk > 0) ? 1u : 0u);
              wgmma_m64n128k16_f16<A_MN ? 1 : 0, B_MN ? 1 : 0>(d, dah, dbl, 1u);
              wgmma_m64n128k16_f16<A_MN ? 1 : 0, B_MN ? 1 : 0>(d, dah, dbh, 1u);
            } else {
              const uint64_t dah = tile_desc<A_MN>(a_hi, kk), dbh = tile_desc<B_MN>(b_hi, kk);
              wgmma_m64n128k16_f16<A_MN ? 1 : 0, B_MN ? 1 : 0>(d, dah, dbh, (kb > kc || kk > 0) ? 1u : 0u);
            }
          }
          wgmma_commit();
          wgmma_wait<1>();                                       // the previous k-block is done ...
          if (held >= 0 && leader) mbar_arrive(&empty[held]);    // ... and this warpgroup no longer reads its slot
          held = stage;
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
          if (kb == kc && g > 0) {
            promote(p, cs_prev);
            if (NSUB > 1 && g == nch) {                          // chunk g - 1 was the last of the first half
              park_acc(park0);
#pragma unroll
              for (int j = 0; j < 64; ++j) acc[j] = 0.f;
            }
          }
        }
        cs_prev = cs;
      };
      // the last chunk, in d: drain, release the last stage, promote, park
      auto finish = [&](float (&d)[64]) {
        wgmma_wait<0>();
        if (leader) mbar_arrive(&empty[held]);
        promote(d, cs_prev);
        if (NSUB > 1) epi_sync();                // both warpgroups are done with the stage ring before it is overwritten
        park_acc(NSUB > 1 ? park1 : park0);
      };
      for (int g = 0;; g += 2) {                 // unrolled by two: d0 / d1 are indexed at compile time
        run_chunk(d0, d1, g);
        if (g + 1 == nchunks) { finish(d0); break; }
        run_chunk(d1, d0, g + 1);
        if (g + 2 == nchunks) { finish(d1); break; }
      }
      epi_sync();

      // ===== epilogue over the parked 128 x BN tile: thread tid handles 4 adjacent columns of rows tid / (BN/4) + k * (1024/BN) =====
      constexpr int CG4 = BN / 4;                  // 4-column groups per row
      constexpr int ROWS_PER_ITER = EPI_THREADS / CG4;
      const int cg = tid % CG4;
      const int c = cg * 4;                        // column inside the tile
      const int col = n0t + c;
      float* const pk = (c < SUB_N ? park0 : park1) + (c & (SUB_N - 1));
      const float alpha = ep.alpha ? __ldg(ep.alpha) : 1.f;
      float bias4[4] = {0.f, 0.f, 0.f, 0.f};
      if (MODE == EPI_FWD && ep.bias) {
        const float inv_alpha = 1.f / alpha;
#pragma unroll
        for (int u = 0; u < 4; ++u) bias4[u] = (col + u < No) ? __ldg(ep.bias + col + u) * inv_alpha : 0.f;
      }
      // ---- ReLU mask of the data-grad (mask = src > 0 or hi > 0): all of this thread's mask entries are loaded before pass 1
      // stores into the parked tile, so the global loads are in flight together instead of one row at a time behind those stores.
      // Bit 4 i + u of mbits: row tid / CG4 + i ROWS_PER_ITER, column col + u.
      constexpr int RPT = BM / ROWS_PER_ITER;      // rows per thread
      const bool has_mask = MODE == EPI_DGRAD && (ep.relu_src || ep.relu_hi);
      uint32_t mbits[RPT / 8];
#pragma unroll
      for (int w = 0; w < RPT / 8; ++w) mbits[w] = 0u;
      if (has_mask && col < No) {
        const int nv = min(4, No - col);
        const bool vec = nv == 4 && (!ep.relu_src || ((ep.ld_relu & 3) == 0 && (reinterpret_cast<uintptr_t>(ep.relu_src) & 15) == 0));
        uint4 raw[RPT];                            // four fp32 words, or four halves in .x / .y
#pragma unroll
        for (int i = 0; i < RPT; ++i) {
          const int row = m0 + tid / CG4 + i * ROWS_PER_ITER;
          raw[i] = make_uint4(0u, 0u, 0u, 0u);
          if (row >= Mo) continue;
          if (!ep.relu_src) {
            const __half* q = ep.relu_hi + (size_t)row * ep.ld_relu_h + col;
            if (vec) {                               // 8-byte aligned: the pitch is a multiple of 8 halves, col of 4
              const uint2 h = __ldg(reinterpret_cast<const uint2*>(q));
              raw[i].x = h.x; raw[i].y = h.y;
            } else {
              const unsigned short* qs = reinterpret_cast<const unsigned short*>(q);
              raw[i].x = __ldg(qs);
              if (nv > 1) raw[i].x |= (uint32_t)__ldg(qs + 1) << 16;
              if (nv > 2) raw[i].y = __ldg(qs + 2);
            }
          } else {
            const float* q = ep.relu_src + (size_t)row * ep.ld_relu + col;
            if (vec) {
              const float4 f = __ldg(reinterpret_cast<const float4*>(q));
              raw[i] = make_uint4(__float_as_uint(f.x), __float_as_uint(f.y), __float_as_uint(f.z), __float_as_uint(f.w));
            } else {
              raw[i].x = __float_as_uint(__ldg(q));
              if (nv > 1) raw[i].y = __float_as_uint(__ldg(q + 1));
              if (nv > 2) raw[i].z = __float_as_uint(__ldg(q + 2));
              if (nv > 3) raw[i].w = __float_as_uint(__ldg(q + 3));     // an unaligned source
            }
          }
        }
#pragma unroll
        for (int i = 0; i < RPT; ++i) {
          float x[4];
          if (!ep.relu_src) {
            const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&raw[i].x));
            const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&raw[i].y));
            x[0] = a.x; x[1] = a.y; x[2] = b.x; x[3] = b.y;
          } else {
            x[0] = __uint_as_float(raw[i].x); x[1] = __uint_as_float(raw[i].y);
            x[2] = __uint_as_float(raw[i].z); x[3] = __uint_as_float(raw[i].w);
          }
#pragma unroll
          for (int u = 0; u < 4; ++u)
            if (x[u] > 0.f) mbits[i / 8] |= 1u << (4 * (i % 8) + u);
        }
      }
      // ---- pass 1: finish the values in place: bias, alpha, activation / ReLU mask; out-of-range entries become exact zeros
      float tmax = 0.f;
#pragma unroll
      for (int i = 0; i < RPT; ++i) {
        const int r = tid / CG4 + i * ROWS_PER_ITER;
        const int row = m0 + r;
        float4* p = reinterpret_cast<float4*>(pk + r * PARK_PITCH);
        float v[4];
        const float4 s = *p;
        v[0] = s.x; v[1] = s.y; v[2] = s.z; v[3] = s.w;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float y = (v[u] + bias4[u]) * alpha;
          if (MODE == EPI_FWD) {
            if (ep.act == GCBF_ACT_RELU) y = fmaxf(y, 0.f);
            else if (ep.act == GCBF_ACT_TANH) y = tanhf(y);
          }
          const bool ok = row < Mo && col + u < No;
          if (has_mask && ok) y = ((mbits[i / 8] >> (4 * (i % 8) + u)) & 1u) ? y : 0.f;
          v[u] = ok ? y : 0.f;
          tmax = fmaxf(tmax, fabsf(v[u]));
        }
        *p = make_float4(v[0], v[1], v[2], v[3]);
      }
      // ---- tile maximum (companion scale) over the 128 x BN tile
      float s_tile = 1.f;
      if (MODE != EPI_WGRAD && ep.out_h) {
        const uint32_t wmax = __reduce_max_sync(0xffffffffu, __float_as_uint(tmax));   // non-negative floats order like uints
        if (lane == 0) red[tid >> 5] = wmax;
        epi_sync();
        uint32_t m = 0;
#pragma unroll
        for (int w = 0; w < EPI_THREADS / 32; ++w) m = max(m, red[w]);
        s_tile = __uint_as_float(scale_bits_from_amax(m));
        if (tid == 0 && m0 < Mo && n0t < No) ep.out_tile_amax[(size_t)(m0 >> 7) * ep.out_amax_stride + (n0t >> 8)] = m;
      }
      // ---- pass 2: outputs
      float out_max = 0.f;
      const bool vec_c = C && (ldc & 3) == 0 && (reinterpret_cast<uintptr_t>(C) & 15) == 0;
      const size_t plane = (size_t)Mo * ep.ld_out_h;
      for (int r = tid / CG4; r < BM; r += ROWS_PER_ITER) {
        const int row = m0 + r;
        if (row >= Mo || col >= No) continue;
        const float4 s = *reinterpret_cast<const float4*>(pk + r * PARK_PITCH);
        const float v[4] = {s.x, s.y, s.z, s.w};
        const int nv = min(4, No - col);
        if (C) {
          float* dst = C + (size_t)blockIdx.y * ep.split_stride + (size_t)row * ldc + col;
          if (ep.accumulate) {
#pragma unroll
            for (int u = 0; u < 4; ++u)
              if (u < nv) { const float o = v[u] + dst[u]; dst[u] = o; out_max = fmaxf(out_max, fabsf(o)); }
          } else if (vec_c && nv == 4) {
            *reinterpret_cast<float4*>(dst) = s;
          } else {
#pragma unroll
            for (int u = 0; u < 4; ++u)
              if (u < nv) dst[u] = v[u];
          }
        }
        if (MODE != EPI_WGRAD && ep.out_h) {
          // hi = fp16(y s), lo = fp16(y s - hi) as in split_h4_kernel
          const float y0 = v[0] * s_tile, y1 = v[1] * s_tile, y2 = v[2] * s_tile, y3 = v[3] * s_tile;
          const __half2 h01 = __floats2half2_rn(y0, y1), h23 = __floats2half2_rn(y2, y3);
          const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
          const __half2 l01 = __floats2half2_rn(__fsub_rn(y0, f01.x), __fsub_rn(y1, f01.y));
          const __half2 l23 = __floats2half2_rn(__fsub_rn(y2, f23.x), __fsub_rn(y3, f23.y));
          __half* dh = ep.out_h + (size_t)row * ep.ld_out_h + col;
          if (nv == 4) {                           // 8-byte aligned: the pitch is a multiple of 8 halves, col of 4
            *reinterpret_cast<uint2*>(dh) = make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
            *reinterpret_cast<uint2*>(dh + plane) = make_uint2(*reinterpret_cast<const uint32_t*>(&l01), *reinterpret_cast<const uint32_t*>(&l23));
          } else {
            const __half hs[4] = {__low2half(h01), __high2half(h01), __low2half(h23), __high2half(h23)};
            const __half ls[4] = {__low2half(l01), __high2half(l01), __low2half(l23), __high2half(l23)};
            for (int u = 0; u < nv; ++u) { dh[u] = hs[u]; dh[plane + u] = ls[u]; }
          }
        }
      }
      if (ep.amax_out && !ep.accumulate) out_max = fmaxf(out_max, tmax);
      // the column sums read what pass 1 of every thread (masking, out-of-range zeros) wrote; with an emitted companion the tile-maximum
      // barrier has already waited for it
      if (MODE == EPI_DGRAD && ep.colsum && !ep.out_h) epi_sync();
      if (MODE == EPI_DGRAD && ep.colsum && tid < BN) {
        // column sums over the tile's rows (the bias gradient of the layer below = colsum of dZ); masked / out-of-range entries are 0
        const float* pc = (tid < SUB_N ? park0 : park1) + (tid & (SUB_N - 1));
        float csum = 0.f;
#pragma unroll 8
        for (int r = 0; r < BM; ++r) csum += pc[r * PARK_PITCH];
        if (n0t + tid < No) ep.colsum[(size_t)(blockIdx.x / tiles_n) * No + n0t + tid] = csum;
      }
      if (ep.amax_out) {
        const uint32_t m = __reduce_max_sync(0xffffffffu, __float_as_uint(out_max));   // non-negative floats order like uints
        if (lane == 0 && m) atomicMax(ep.amax_out, m);
      }
    }
  }
}
// ---- amax and the [hi | lo] split ------------------------------------------------------------------------------
// max|x| over a strided [rows, cols] fp32 matrix -> atomicMax on the float bits (non-negative floats order like uints)
__global__ void amax_kernel(const float* __restrict__ src, int ld, int rows, int cols, uint32_t* __restrict__ slot, int vec4) {
  float m = 0.f;
  if (vec4) {
    const int w = cols >> 2;
    for (int r = blockIdx.x; r < rows; r += gridDim.x) {
      const float4* p = reinterpret_cast<const float4*>(src + (size_t)r * ld);
      for (int c = threadIdx.x; c < w; c += blockDim.x) {
        const float4 x = __ldg(p + c);
        m = fmaxf(fmaxf(m, fmaxf(fabsf(x.x), fabsf(x.y))), fmaxf(fabsf(x.z), fabsf(x.w)));
      }
    }
  } else {
    for (int r = blockIdx.x; r < rows; r += gridDim.x)
      for (int c = threadIdx.x; c < cols; c += blockDim.x) m = fmaxf(m, fabsf(__ldg(src + (size_t)r * ld + c)));
  }
  const uint32_t w = __reduce_max_sync(0xffffffffu, __float_as_uint(m));
  __shared__ uint32_t part[32];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = w;
  __syncthreads();
  if (threadIdx.x < 32) {
    uint32_t v = threadIdx.x < (blockDim.x >> 5) ? part[threadIdx.x] : 0u;
    v = __reduce_max_sync(0xffffffffu, v);
    if (threadIdx.x == 0 && v) atomicMax(slot, v);
  }
}

// dst planes: hi at dst, lo at dst + rows*ld_h (halves); element (r, c) of the fp32 source -> same (r, c).  Each thread
// converts 2 adjacent columns; a block walks `strip` rows so the optional column sums (bias gradient = colsum of dZ,
// reference autograd of nn.Linear) need one partial per column per block.
constexpr int SPLIT_ROWS = 64;
__global__ void split_h_kernel(const float* __restrict__ src, int ld, int rows, int cols, const uint32_t* __restrict__ amax,
                               __half* __restrict__ dst, int ld_h, float* __restrict__ colsum) {
  const float s = __uint_as_float(scale_bits_from_amax(__ldg(amax)));
  const int c = (blockIdx.x * 32 + threadIdx.x) * 2;
  const int r0 = blockIdx.y * SPLIT_ROWS;
  const size_t plane = (size_t)rows * ld_h;
  float s0 = 0.f, s1 = 0.f;
  if (c < cols) {
    const bool pair = (c + 1 < cols);
    const int r1 = min(rows, r0 + SPLIT_ROWS);
    for (int r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
      const float* p = src + (size_t)r * ld + c;
      const float x0 = __ldg(p), x1 = pair ? __ldg(p + 1) : 0.f;
      const float y0 = x0 * s, y1 = x1 * s;
      const __half2 hi = __floats2half2_rn(y0, y1);
      const float2 hf = __half22float2(hi);
      const __half2 lo = __floats2half2_rn(__fsub_rn(y0, hf.x), __fsub_rn(y1, hf.y));
      __half* d = dst + (size_t)r * ld_h + c;
      if (pair) {
        *reinterpret_cast<__half2*>(d) = hi;
        *reinterpret_cast<__half2*>(d + plane) = lo;
      } else {
        d[0] = __low2half(hi);
        d[plane] = __low2half(lo);
      }
      s0 += x0; s1 += x1;
    }
  }
  if (colsum) {
    __shared__ float red[8][64];
    red[threadIdx.y][2 * threadIdx.x] = s0;
    red[threadIdx.y][2 * threadIdx.x + 1] = s1;
    __syncthreads();
    if (threadIdx.y == 0) {
      float t0 = 0.f, t1 = 0.f;
#pragma unroll
      for (int y = 0; y < 8; ++y) { t0 += red[y][2 * threadIdx.x]; t1 += red[y][2 * threadIdx.x + 1]; }
      if (c < cols) colsum[(size_t)blockIdx.y * cols + c] = t0;          // this row strip's partials ([strips][cols])
      if (c + 1 < cols) colsum[(size_t)blockIdx.y * cols + c + 1] = t1;
    }
  }
}

// the same split for the aligned case (cols and pitch multiples of 4, 16-byte aligned source): 4 columns per thread,
// one 16-byte load and one 8-byte store per plane per row, 4 rows in flight
__device__ __forceinline__ void split4(const float4 x, float s, uint2& hi, uint2& lo) {
  const float y0 = x.x * s, y1 = x.y * s, y2 = x.z * s, y3 = x.w * s;
  const __half2 h01 = __floats2half2_rn(y0, y1), h23 = __floats2half2_rn(y2, y3);
  const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
  const __half2 l01 = __floats2half2_rn(__fsub_rn(y0, f01.x), __fsub_rn(y1, f01.y));
  const __half2 l23 = __floats2half2_rn(__fsub_rn(y2, f23.x), __fsub_rn(y3, f23.y));
  hi.x = *reinterpret_cast<const uint32_t*>(&h01); hi.y = *reinterpret_cast<const uint32_t*>(&h23);
  lo.x = *reinterpret_cast<const uint32_t*>(&l01); lo.y = *reinterpret_cast<const uint32_t*>(&l23);
}

__global__ void __launch_bounds__(256) split_h4_kernel(const float* __restrict__ src, int ld, int rows, int cols,
                                                       const uint32_t* __restrict__ amax, __half* __restrict__ dst, int ld_h,
                                                       float* __restrict__ colsum) {
  const float s = __uint_as_float(scale_bits_from_amax(__ldg(amax)));
  const int c = (blockIdx.x * 32 + threadIdx.x) * 4;
  const int r0 = blockIdx.y * SPLIT_ROWS;
  const size_t plane = (size_t)rows * ld_h;
  float cs[4] = {0.f, 0.f, 0.f, 0.f};
  if (c < cols) {
    const int r1 = min(rows, r0 + SPLIT_ROWS);
    for (int r = r0 + threadIdx.y; r < r1; r += 32) {        // 4 rows (8 apart) per iteration
      float4 x[4];
#pragma unroll
      for (int u = 0; u < 4; ++u)
        x[u] = (r + 8 * u < r1) ? __ldg(reinterpret_cast<const float4*>(src + (size_t)(r + 8 * u) * ld + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (r + 8 * u < r1) {
          uint2 hi, lo;
          split4(x[u], s, hi, lo);
          __half* d = dst + (size_t)(r + 8 * u) * ld_h + c;
          *reinterpret_cast<uint2*>(d) = hi;
          *reinterpret_cast<uint2*>(d + plane) = lo;
          cs[0] += x[u].x; cs[1] += x[u].y; cs[2] += x[u].z; cs[3] += x[u].w;
        }
      }
    }
  }
  if (colsum) {
    __shared__ float red[8][128];
#pragma unroll
    for (int j = 0; j < 4; ++j) red[threadIdx.y][4 * threadIdx.x + j] = cs[j];
    __syncthreads();
    if (threadIdx.y < 4) {                                   // 4 x 32 threads reduce the 128 columns of the block
      const int col = threadIdx.y * 32 + threadIdx.x;
      float t = 0.f;
#pragma unroll
      for (int y = 0; y < 8; ++y) t += red[y][col];
      const int gc = blockIdx.x * 128 + col;
      if (gc < cols) colsum[(size_t)blockIdx.y * cols + gc] = t;        // this row strip's partials ([strips][cols])
    }
  }
}

// ---- batched amax + split: the companions of all (stale) weight matrices of a net in two launches -------------------------
constexpr int kSplitMaxBatch = 16;
struct SplitBatch {
  const float* src[kSplitMaxBatch];
  uint32_t* amax[kSplitMaxBatch];
  __half* dst[kSplitMaxBatch];
  int ld[kSplitMaxBatch], rows[kSplitMaxBatch], cols[kSplitMaxBatch], ld_h[kSplitMaxBatch];
};

__global__ void __launch_bounds__(256) amax_batched_kernel(const __grid_constant__ SplitBatch b) {
  // one warp per row (8 rows per block), 16-byte loads where the matrix allows them; blocks beyond a matrix's rows exit
  const int t = blockIdx.z;
  const int ld = b.ld[t], rows = b.rows[t], cols = b.cols[t];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* __restrict__ src = b.src[t];
  const bool vec = ((cols & 3) == 0 && (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0);
  float m = 0.f;
  for (int r = blockIdx.x * 8 + warp; r < rows; r += gridDim.x * 8) {
    const float* row = src + (size_t)r * ld;
    if (vec) {
      const float4* p = reinterpret_cast<const float4*>(row);
      for (int c = lane; c < (cols >> 2); c += 32) {
        const float4 x = __ldg(p + c);
        m = fmaxf(fmaxf(m, fmaxf(fabsf(x.x), fabsf(x.y))), fmaxf(fabsf(x.z), fabsf(x.w)));
      }
    } else {
      for (int c = lane; c < cols; c += 32) m = fmaxf(m, fabsf(__ldg(row + c)));
    }
  }
  const uint32_t w = __reduce_max_sync(0xffffffffu, __float_as_uint(m));
  __shared__ uint32_t part[8];
  if (lane == 0) part[warp] = w;
  __syncthreads();
  if (threadIdx.x < 32) {
    uint32_t v = threadIdx.x < 8 ? part[threadIdx.x] : 0u;
    v = __reduce_max_sync(0xffffffffu, v);
    if (threadIdx.x == 0 && v) atomicMax(b.amax[t], v);
  }
}

__global__ void __launch_bounds__(256) split_batched_kernel(const __grid_constant__ SplitBatch b) {
  const int t = blockIdx.z;
  const int ld = b.ld[t], rows = b.rows[t], cols = b.cols[t], ld_h = b.ld_h[t];
  const int c = (blockIdx.x * 32 + threadIdx.x) * 2;
  const int r0 = blockIdx.y * SPLIT_ROWS;
  if (c >= cols || r0 >= rows) return;
  const float* __restrict__ src = b.src[t];
  __half* __restrict__ dst = b.dst[t];
  const float s = __uint_as_float(scale_bits_from_amax(*b.amax[t]));
  const size_t plane = (size_t)rows * ld_h;
  const bool pair = (c + 1 < cols);
  const int r1 = min(rows, r0 + SPLIT_ROWS);
  for (int r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
    const float* p = src + (size_t)r * ld + c;
    const float y0 = __ldg(p) * s, y1 = pair ? __ldg(p + 1) * s : 0.f;
    const __half2 hi = __floats2half2_rn(y0, y1);
    const float2 hf = __half22float2(hi);
    const __half2 lo = __floats2half2_rn(__fsub_rn(y0, hf.x), __fsub_rn(y1, hf.y));
    __half* d = dst + (size_t)r * ld_h + c;
    if (pair) {
      *reinterpret_cast<__half2*>(d) = hi;
      *reinterpret_cast<__half2*>(d + plane) = lo;
    } else {
      d[0] = __low2half(hi);
      d[plane] = __low2half(lo);
    }
  }
}

// ---- host side -----------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && p) fn = (EncodeTiledFn)p;
  }
  return fn;
}

// one fp16 plane [rows][cols] (pitch ld_h halves).  K-major use: box {BK cols, tile_rows rows}, SWIZZLE_64B;
// MN-major use: box {64 cols, BK rows}, SWIZZLE_128B.
static int make_map(CUtensorMap* map, const __half* base, int rows, int cols, int ld_h, bool mn_major, int tile_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return GCBF_E_CUDA; }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld_h * 2};
  cuuint32_t box[2] = {(cuuint32_t)(mn_major ? MN_BOX : BK), (cuuint32_t)(mn_major ? BK : tile_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, mn_major ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) rows=%d cols=%d ld=%d mn=%d", (int)r, rows, cols, ld_h, (int)mn_major);
    return GCBF_E_CUDA;
  }
  return GCBF_OK;
}

// wgmma launches per product count ([0]: 3xFP16, [1]: one product), read by gcbf_tc_launch_count: which kernels a pass really ran
static std::atomic<long long> g_tc_launches[2];

static bool g_env_read = false;
// k-blocks per promotion chunk.  The tensor core TRUNCATES its fp32 accumulator on every MMA (tools/acc_probe.py): the bias grows with the
// number of MMAs accumulated before the chunk sum is promoted to registers with round-to-nearest.  4 k-blocks = 128 K-elements = 24 MMAs
// per chunk (GCBF_TC_KCH overrides it, 1..8)
static int g_kch = 4;
static int g_kch_dgrad = 8;     // data-grad products with per-tensor operands keep 256-element chunks: their result is a gradient (parity bar: 2e-2
                                // of the gradient norm), the forward's 1e-5 bar on h / u does not depend on them.  GCBF_TC_KCH_DGRAD

// companion operand as the GEMM sees it: plane [rows][cols]; K-major: rows = output index, cols = contraction;
// MN-major: rows = contraction, cols = output index
struct Operand {
  const __half* hi; int rows; int cols; int ld_h; bool mn_major;
  const __half* lo() const { return hi + (size_t)rows * ld_h; }
};
// companion the epilogue writes (tile-scaled): planes [rows][cols] like an Operand, plus the tile-maxima array
struct OutH {
  __half* hi; int rows; int cols; int ld_h; uint32_t* tile_amax; int amax_stride;
};

template <int BN, bool A_MN, bool B_MN, int P>
static int launch(const Operand& A, const Operand& B, float* C, int ldc, int Mo, int No, int Kc, int splits, EpiParams ep,
                  const OutH* oh, cudaStream_t st) {
  if (!g_env_read) {
    const char* kc = getenv("GCBF_TC_KCH");
    if (kc && atoi(kc) >= 1 && atoi(kc) <= KCH_MAX) g_kch = atoi(kc);
    const char* kd = getenv("GCBF_TC_KCH_DGRAD");
    if (kd && atoi(kd) >= 1 && atoi(kd) <= KCH_MAX) g_kch_dgrad = atoi(kd);
    if (kc && !kd) g_kch_dgrad = g_kch > 4 ? g_kch : g_kch_dgrad;
    g_env_read = true;
  }
  if ((ep.a_sr || ep.a_sc || ep.b_sr || ep.b_sc) && g_kch > 4) { set_error("tile-scaled operands need promotion chunks of <= 128 K-elements (GCBF_TC_KCH <= 4)"); return GCBF_E_UNSUPPORTED; }
  if constexpr (BN != 256 || A_MN) {
    if (oh || ep.colsum) { set_error("companion emission / column sums need a 256-wide forward or data-grad launch"); return GCBF_E_UNSUPPORTED; }
  }
  CUtensorMap mah, mal, mbh, mbl;
  if (int rc = make_map(&mah, A.hi, A.rows, A.cols, A.ld_h, A_MN, BM)) return rc;
  if (int rc = make_map(&mbh, B.hi, B.rows, B.cols, B.ld_h, B_MN, SUB_N)) return rc;
  if (P == 3) {
    if (int rc = make_map(&mal, A.lo(), A.rows, A.cols, A.ld_h, A_MN, BM)) return rc;
    if (int rc = make_map(&mbl, B.lo(), B.rows, B.cols, B.ld_h, B_MN, SUB_N)) return rc;
  } else {
    mal = mah; mbl = mbh;                   // not read by the one-product kernel
  }
  if (oh) {
    ep.out_h = oh->hi; ep.ld_out_h = oh->ld_h; ep.out_tile_amax = oh->tile_amax; ep.out_amax_stride = oh->amax_stride;
  }
  static bool attr_set = false;
  if (!attr_set) {
    GCBF_CUDA_OK(cudaFuncSetAttribute(gemm_h_kernel<BN, A_MN, B_MN, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    attr_set = true;
  }
  const int tiles_m = ceil_div(Mo, BM), tiles_n = ceil_div(No, BN);
  const int kblocks = ceil_div(Kc, BK);
  // data-grad: a K-major tile-scaled A (scale tiles 256 contraction elements wide) is compatible with 256-element chunks; an MN-major
  // tile-scaled operand (scale rows of 128 contraction elements) is not
  const int kch = (!A_MN && B_MN && !(ep.b_sr || ep.b_sc)) ? g_kch_dgrad : g_kch;
  // chunks of kch k-blocks must not straddle splits (tile-scaled operands: a chunk lies inside one scale tile)
  const int kps = ceil_div(ceil_div(kblocks, splits), kch) * kch;
  const int nsplit = ceil_div(kblocks, kps);
  // split-K slices and per-row-tile column sums go to scratch and are summed in a fixed order afterwards (deterministic results)
  float* part = nullptr;
  float* colsum_part = nullptr;
  float* const colsum = ep.colsum;
  const int accumulate = ep.accumulate;
  if (nsplit > 1) {
    GCBF_CUDA_OK(scratch_alloc((void**)&part, (size_t)nsplit * Mo * No * 4, st));
    ep.split_stride = (size_t)Mo * No;
    ep.accumulate = 0;
  }
  if (colsum) {
    GCBF_CUDA_OK(scratch_alloc((void**)&colsum_part, (size_t)tiles_m * No * 4, st));
    ep.colsum = colsum_part;
  }
  gemm_h_kernel<BN, A_MN, B_MN, P><<<dim3(tiles_m * tiles_n, nsplit), NUM_THREADS, SMEM_BYTES, st>>>(mah, mal, mbh, mbl, part ? part : C,
                                                                                                    part ? No : ldc, Mo, No, tiles_n, kps,
                                                                                                    kblocks, kch, ep);
  GCBF_LAUNCH_OK();
  g_tc_launches[P == 1 ? 1 : 0].fetch_add(1, std::memory_order_relaxed);
  if (part) {
    GCBF_CUDA_OK(add_partials(part, nsplit, Mo, No, C, ldc, accumulate, st));
    GCBF_CUDA_OK(scratch_free(part, st));
  }
  if (colsum_part) {
    GCBF_CUDA_OK(add_partials(colsum_part, tiles_m, 1, No, colsum, No, 1, st));
    GCBF_CUDA_OK(scratch_free(colsum_part, st));
  }
  return GCBF_OK;
}

// products per k-slice chosen at run time: 3 (3xFP16) or 1 (fp16 operands, the hi planes only)
template <int BN, bool A_MN, bool B_MN>
static int launch_p(int products, const Operand& A, const Operand& B, float* C, int ldc, int Mo, int No, int Kc, int splits,
                    const EpiParams& ep, const OutH* oh, cudaStream_t st) {
  return products == 1 ? launch<BN, A_MN, B_MN, 1>(A, B, C, ldc, Mo, No, Kc, splits, ep, oh, st)
                       : launch<BN, A_MN, B_MN, 3>(A, B, C, ldc, Mo, No, Kc, splits, ep, oh, st);
}

static int check_plane(const void* p, int ld_h, const char* what) {
  if (!p || (reinterpret_cast<uintptr_t>(p) & 15) || (ld_h & 7)) {
    set_error("%s: fp16 companion must be 16-byte aligned with a pitch that is a multiple of 8 halves (ptr=%p ld=%d)", what, p, ld_h);
    return GCBF_E_INVALID;
  }
  return GCBF_OK;
}

}  // namespace th
}  // namespace gcbf

using namespace gcbf;

// ---- C ABI ------------------------------------------------------------------------------------------------------
extern "C" int gcbf_amax_f32(const float* src, int ld, int rows, int cols, void* amax_slot, int accumulate, void* stream) {
  GCBF_REQUIRE(amax_slot && rows >= 0 && cols >= 0 && ld >= cols, "gcbf_amax_f32: bad arguments rows=%d cols=%d ld=%d", rows, cols, ld);
  cudaStream_t st = as_stream(stream);
  if (!accumulate) GCBF_CUDA_OK(cudaMemsetAsync(amax_slot, 0, 4, st));
  if (rows == 0 || cols == 0) return GCBF_OK;
  GCBF_REQUIRE(src, "gcbf_amax_f32: null src");
  const int vec4 = ((cols & 3) == 0 && (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0) ? 1 : 0;
  const int work = vec4 ? cols / 4 : cols;
  const int threads = work >= 256 ? 256 : (work >= 128 ? 128 : 64);
  const int blocks = (int)imin64(rows, (int64_t)kNumSMs * (2048 / threads));
  th::amax_kernel<<<blocks, threads, 0, st>>>(src, ld, rows, cols, reinterpret_cast<uint32_t*>(amax_slot), vec4);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

extern "C" int gcbf_split_f16(const float* src, int ld, int rows, int cols, const void* amax_slot, void* dst, int ld_h,
                              float* colsum, int colsum_accumulate, void* stream) {
  GCBF_REQUIRE(amax_slot && dst && rows >= 0 && cols >= 0 && ld >= cols && ld_h >= cols, "gcbf_split_f16: bad arguments rows=%d cols=%d", rows, cols);
  if (int rc = th::check_plane(dst, ld_h, "gcbf_split_f16")) return rc;
  cudaStream_t st = as_stream(stream);
  if (colsum && !colsum_accumulate) GCBF_CUDA_OK(cudaMemsetAsync(colsum, 0, (size_t)cols * 4, st));
  if (rows == 0 || cols == 0) return GCBF_OK;
  GCBF_REQUIRE(src, "gcbf_split_f16: null src");
  dim3 block(32, 8);
  const int strips = ceil_div(rows, th::SPLIT_ROWS);
  float* part = nullptr;      // column sums: one row of partials per row strip, summed in a fixed order below
  if (colsum) GCBF_CUDA_OK(scratch_alloc((void**)&part, (size_t)strips * cols * 4, st));
  if ((cols & 3) == 0 && (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
    dim3 grid(ceil_div(cols, 128), strips);
    th::split_h4_kernel<<<grid, block, 0, st>>>(src, ld, rows, cols, reinterpret_cast<const uint32_t*>(amax_slot),
                                               reinterpret_cast<__half*>(dst), ld_h, part);
  } else {
    dim3 grid(ceil_div(cols, 64), strips);
    th::split_h_kernel<<<grid, block, 0, st>>>(src, ld, rows, cols, reinterpret_cast<const uint32_t*>(amax_slot),
                                              reinterpret_cast<__half*>(dst), ld_h, part);
  }
  GCBF_LAUNCH_OK();
  if (part) {
    GCBF_CUDA_OK(add_partials(part, strips, 1, cols, colsum, cols, 1, st));
    GCBF_CUDA_OK(scratch_free(part, st));
  }
  return GCBF_OK;
}

// gcbf_amax_f32 + gcbf_split_f16 for `count` matrices (HOST array of descriptors) in two launches per 16 matrices: the
// weights of a net after an optimizer step.  Same arithmetic per matrix, so the companions are bit-identical.
extern "C" int gcbf_amax_split_batched(const gcbf_split_desc* descs, int count, void* stream) {
  GCBF_REQUIRE(descs && count >= 0, "gcbf_amax_split_batched: bad arguments");
  cudaStream_t st = as_stream(stream);
  for (int base = 0; base < count; base += th::kSplitMaxBatch) {
    const int nb = min(th::kSplitMaxBatch, count - base);
    th::SplitBatch b{};
    int max_rows = 0, max_cols = 0;
    for (int i = 0; i < nb; ++i) {
      const gcbf_split_desc& d = descs[base + i];
      GCBF_REQUIRE(d.src && d.amax_slot && d.dst && d.rows > 0 && d.cols > 0 && d.ld >= d.cols && d.ld_h >= d.cols,
                   "gcbf_amax_split_batched: descriptor %d", base + i);
      if (int rc = th::check_plane(d.dst, d.ld_h, "gcbf_amax_split_batched")) return rc;
      b.src[i] = d.src; b.amax[i] = reinterpret_cast<uint32_t*>(d.amax_slot); b.dst[i] = reinterpret_cast<__half*>(d.dst);
      b.ld[i] = d.ld; b.rows[i] = d.rows; b.cols[i] = d.cols; b.ld_h[i] = d.ld_h;
      max_rows = max(max_rows, d.rows); max_cols = max(max_cols, d.cols);
      GCBF_CUDA_OK(cudaMemsetAsync(d.amax_slot, 0, 4, st));
    }
    th::amax_batched_kernel<<<dim3(min(ceil_div(max_rows, 8), 8 * kNumSMs), 1, nb), 256, 0, st>>>(b);
    GCBF_LAUNCH_OK();
    th::split_batched_kernel<<<dim3(ceil_div(max_cols, 64), ceil_div(max_rows, th::SPLIT_ROWS), nb), dim3(32, 8), 0, st>>>(b);
    GCBF_LAUNCH_OK();
  }
  return GCBF_OK;
}

extern "C" long long gcbf_tc_launch_count(int products, int reset) {
  if (products != 1 && products != 3) { set_error("gcbf_tc_launch_count: products %d (3 or 1)", products); return -1; }
  std::atomic<long long>& c = th::g_tc_launches[products == 1 ? 1 : 0];
  return reset ? c.exchange(0) : c.load();
}

extern "C" int gcbf_linear_h_supported(int M, int N, int K) {
  // the rule the host mirror applies per layer (forward, data-grad and weight-grad alike): enough rows to fill 128-row tiles,
  // both feature dimensions wide enough to be a tile / a contraction, and enough work to amortise the split pass
  return (M >= 256 && N >= 96 && K >= 96 && (long long)M * N * K >= (1ll << 24)) ? 1 : 0;
}

static int check_h16(const gcbf_h16* h, const char* what, int rows, int cols) {
  if (!h || !h->buf || !h->amax || h->rows != rows || h->cols != cols || h->ld < cols) {
    set_error("%s: companion descriptor (expected [%d x %d])", what, rows, cols);
    return GCBF_E_INVALID;
  }
  return th::check_plane(h->buf, h->ld, what);
}

// Y[M,N] = act(alpha * X W^T + bias): A = X companion [M][K] (K-major), B = W companion [N][K] (K-major, per-tensor scale).
// products: 3 (3xFP16) or 1 (fp16: the hi planes only; the companions keep their [hi|lo] format)
extern "C" int gcbf_linear_fwd_h(const gcbf_h16* X, const gcbf_h16* W, const float* bias, const float* inv_sigma, int act, float* Y, int ldy,
                                 const gcbf_h16* Yh, void* out_amax, int M, int N, int K, void* stream, int products) {
  GCBF_REQUIRE(M > 0 && N > 0 && K > 0 && (Y || Yh) && (!Y || ldy >= N), "gcbf_linear_fwd_h: bad arguments M=%d N=%d K=%d", M, N, K);
  GCBF_REQUIRE(products == 3 || products == 1, "gcbf_linear_fwd_h: products %d (3 or 1)", products);
  if (int rc = check_h16(X, "gcbf_linear_fwd_h X", M, K)) return rc;
  if (int rc = check_h16(W, "gcbf_linear_fwd_h W", N, K)) return rc;
  GCBF_REQUIRE(W->amax_row_stride == 0 && W->amax_col_stride == 0, "gcbf_linear_fwd_h: the weight companion must be per-tensor scaled");
  cudaStream_t st = as_stream(stream);
  th::EpiParams ep{};
  ep.mode = th::EPI_FWD; ep.alpha = inv_sigma; ep.bias = bias; ep.act = act;
  ep.amax_a = reinterpret_cast<const uint32_t*>(X->amax); ep.a_sr = X->amax_row_stride; ep.a_sc = X->amax_col_stride;
  ep.amax_b = reinterpret_cast<const uint32_t*>(W->amax);
  ep.amax_out = reinterpret_cast<uint32_t*>(out_amax);
  if (out_amax) GCBF_CUDA_OK(cudaMemsetAsync(out_amax, 0, 4, st));
  th::OutH oh{};
  if (Yh) {
    if (int rc = check_h16(Yh, "gcbf_linear_fwd_h Yh", M, N)) return rc;
    GCBF_REQUIRE(N > 128 && Yh->amax_row_stride == ceil_div(N, 256) && Yh->amax_col_stride == 1, "gcbf_linear_fwd_h: emitted companions are tile-scaled (N > 128, amax strides (ceil(N/256), 1))");
    oh = th::OutH{reinterpret_cast<__half*>(Yh->buf), M, N, Yh->ld, reinterpret_cast<uint32_t*>(Yh->amax), Yh->amax_row_stride};
  }
  th::Operand A{reinterpret_cast<const __half*>(X->buf), M, K, X->ld, false}, B{reinterpret_cast<const __half*>(W->buf), N, K, W->ld, false};
  return (N > 128) ? th::launch_p<256, false, false>(products, A, B, Y, ldy, M, N, K, 1, ep, Yh ? &oh : nullptr, st)
                   : th::launch_p<128, false, false>(products, A, B, Y, ldy, M, N, K, 1, ep, nullptr, st);
}

// dX[M,K] (+)= alpha * dZ W (* relu mask): A = dZ companion [M][N] (K-major: contraction over N), B = W companion [N][K] (MN-major)
extern "C" int gcbf_linear_bwd_data_h(const gcbf_h16* dZ, const gcbf_h16* W, const float* inv_sigma, const float* relu_src, int ld_relu,
                                      const gcbf_h16* relu_h, float* dX, int lddx, int accumulate, const gcbf_h16* dXh, float* colsum,
                                      void* out_amax, int M, int N, int K, void* stream, int products) {
  GCBF_REQUIRE(M > 0 && N > 0 && K > 0 && (dX || dXh) && (!dX || lddx >= K), "gcbf_linear_bwd_data_h: bad arguments M=%d N=%d K=%d", M, N, K);
  GCBF_REQUIRE(products == 3 || products == 1, "gcbf_linear_bwd_data_h: products %d (3 or 1)", products);
  GCBF_REQUIRE(!relu_src || ld_relu >= K, "gcbf_linear_bwd_data_h: ld_relu");
  GCBF_REQUIRE(!(relu_src && relu_h) && !(accumulate && (dXh || colsum)), "gcbf_linear_bwd_data_h: conflicting options");
  if (int rc = check_h16(dZ, "gcbf_linear_bwd_data_h dZ", M, N)) return rc;
  if (int rc = check_h16(W, "gcbf_linear_bwd_data_h W", N, K)) return rc;
  GCBF_REQUIRE(W->amax_row_stride == 0 && W->amax_col_stride == 0, "gcbf_linear_bwd_data_h: the weight companion must be per-tensor scaled");
  if (relu_h) { if (int rc = check_h16(relu_h, "gcbf_linear_bwd_data_h relu_h", M, K)) return rc; }
  cudaStream_t st = as_stream(stream);
  th::EpiParams ep{};
  ep.mode = th::EPI_DGRAD; ep.alpha = inv_sigma; ep.relu_src = relu_src; ep.ld_relu = ld_relu; ep.accumulate = accumulate;
  if (relu_h) { ep.relu_hi = reinterpret_cast<const __half*>(relu_h->buf); ep.ld_relu_h = relu_h->ld; }
  ep.amax_a = reinterpret_cast<const uint32_t*>(dZ->amax); ep.a_sr = dZ->amax_row_stride; ep.a_sc = dZ->amax_col_stride;
  ep.amax_b = reinterpret_cast<const uint32_t*>(W->amax);
  ep.amax_out = reinterpret_cast<uint32_t*>(out_amax);
  ep.colsum = colsum;
  if (out_amax) GCBF_CUDA_OK(cudaMemsetAsync(out_amax, 0, 4, st));
  th::OutH oh{};
  if (dXh) {
    if (int rc = check_h16(dXh, "gcbf_linear_bwd_data_h dXh", M, K)) return rc;
    GCBF_REQUIRE(K > 128 && dXh->amax_row_stride == ceil_div(K, 256) && dXh->amax_col_stride == 1, "gcbf_linear_bwd_data_h: emitted companions are tile-scaled (K > 128, amax strides (ceil(K/256), 1))");
    oh = th::OutH{reinterpret_cast<__half*>(dXh->buf), M, K, dXh->ld, reinterpret_cast<uint32_t*>(dXh->amax), dXh->amax_row_stride};
  }
  th::Operand A{reinterpret_cast<const __half*>(dZ->buf), M, N, dZ->ld, false}, B{reinterpret_cast<const __half*>(W->buf), N, K, W->ld, true};
  return (K > 128) ? th::launch_p<256, false, true>(products, A, B, dX, lddx, M, K, N, 1, ep, dXh ? &oh : nullptr, st)
                   : th::launch_p<128, false, true>(products, A, B, dX, lddx, M, K, N, 1, ep, nullptr, st);
}

// dW[N,K] (+)= alpha * dZ^T X: A = dZ companion [M][N] (MN-major), B = X companion [M][K] (MN-major); contraction over M
extern "C" int gcbf_linear_bwd_weight_h(const gcbf_h16* dZ, const gcbf_h16* X, const float* inv_sigma, float* dW, int lddw, int accumulate,
                                        int M, int N, int K, void* stream, int products) {
  GCBF_REQUIRE(M > 0 && N > 0 && K > 0 && lddw >= K && dW, "gcbf_linear_bwd_weight_h: bad arguments M=%d N=%d K=%d", M, N, K);
  GCBF_REQUIRE(products == 3 || products == 1, "gcbf_linear_bwd_weight_h: products %d (3 or 1)", products);
  if (int rc = check_h16(dZ, "gcbf_linear_bwd_weight_h dZ", M, N)) return rc;
  if (int rc = check_h16(X, "gcbf_linear_bwd_weight_h X", M, K)) return rc;
  cudaStream_t st = as_stream(stream);
  th::EpiParams ep{};
  ep.mode = th::EPI_WGRAD; ep.alpha = inv_sigma; ep.accumulate = accumulate;
  ep.amax_a = reinterpret_cast<const uint32_t*>(dZ->amax); ep.a_sr = dZ->amax_row_stride; ep.a_sc = dZ->amax_col_stride;
  ep.amax_b = reinterpret_cast<const uint32_t*>(X->amax); ep.b_sr = X->amax_row_stride; ep.b_sc = X->amax_col_stride;
  const int BN = (K > 128) ? 256 : 128;
  const int tiles = ceil_div(N, th::BM) * ceil_div(K, BN);
  int splits = 1;
  if (tiles < kNumSMs) splits = max(1, min(ceil_div(M, 256), kNumSMs / tiles));
  th::Operand A{reinterpret_cast<const __half*>(dZ->buf), M, N, dZ->ld, true}, B{reinterpret_cast<const __half*>(X->buf), M, K, X->ld, true};
  return (BN == 256) ? th::launch_p<256, true, true>(products, A, B, dW, lddw, N, K, M, splits, ep, nullptr, st)
                     : th::launch_p<128, true, true>(products, A, B, dW, lddw, N, K, M, splits, ep, nullptr, st);
}
