// 3x3 / 1x1 convolution as an implicit GEMM on the sm_90a tensor cores (wgmma).
//
// Replaces, for the U-Net of lungmask/resunet.py, every Conv2d(3x3,pad 1)+ReLU+BatchNorm2d pair
// (resunet.py:93-105), the decoder's 1x1 convolutions (resunet.py:133, evaluated below the upsample),
// the 2x2 average pool (resunet.py:64, fused as an epilogue), the channel concat (resunet.py:147,
// "virtual": the K loop walks two tensor maps) and the head 1x1 + LogSoftmax + argmax
// (resunet.py:69-70, mask.py:184-186, fused into the last convolution's epilogue).
//
// GEMM view: M = 128 output pixels (a 16-row x 8-column patch of one image), N = BN output channels,
// K = taps * Cin walked in k-blocks of BK input channels of one filter tap, BK = one 128-byte row of the operand
// format (conv_tc.cuh: 64 fp16 or 32 tf32 channels).
//   * A operand: ONE 5-D TMA box per BK-channel block - the patch plus its one-pixel halo,
//     (BK ch, 10 x, 18 y, 2 planes, 1 image) = 180 rows of 128 B per plane - serves all nine taps: the tap
//     (dy,dx) view is the same shared-memory tile entered at row (dy+1)*10 + (dx+1) with an 8-row-group
//     stride of 10 rows (wgmma shared-memory descriptors allow that: the 128B swizzle is a function of the
//     absolute shared-memory address).  TMA zero-fills outside the image, which IS the convolution's zero padding.
//   * B operand: one 4-D TMA box (BK cin, BN cout, 1 tap, 2 planes) per k-block, into a ring of STAGES.
//   * both land 128B-swizzled, K-major, i.e. in the canonical wgmma shared-memory layout.
//   * fp32-class accuracy from 11-bit tensor-core operands: every fp32 value is pre-split into a hi and a lo plane
//     (fp16 hi + fp16 lo * 2^-11 by default, tf32 hi + tf32 lo with LM_OPERAND_F16=0) and each k-step computes
//     hi*hi, hi*lo and lo*hi - three exact products - as three N = BN wgmmas, hi*hi into one accumulator and both
//     corrections into another.  (One N = 2*BN wgmma over [hi*hi | hi*lo] would save an instruction, but its
//     accumulator overlaps the lo*hi one and ptxas then serialises every wgmma of the kernel.)  The tensor
//     core's fp32 accumulation does not round to nearest, so the dominant hi*hi sum is kept apart from the
//     2^-11-times-smaller corrections: only `chunk_kb` k-blocks of hi*hi are accumulated by the tensor core before
//     the partial sum is added, round-to-nearest, into a separate fp32 register sum.  The corrections accumulate in
//     the tensor core for the whole tile.
//   * persistent CTAs (one per SM), warp-specialised: warp 0 is the TMA producer, warpgroups 1 and 2 are consumers
//     that each own 64 rows of the tile (image rows 0-7 / 8-15 of the patch): they issue the wgmmas, drain the
//     chunks and run the epilogue of their rows from the accumulator registers.  Split-plane outputs (fp16 build) are
//     staged in the tile's last activation buffer and written by warp 1, the storer, with TMA stores, so that the
//     consumers go back to the wgmmas instead of waiting for scattered global stores to drain.
//   * the 3x3 layers with 64 output channels run conv_cm64_kernel (below) unless ConvParams::conv64_cm is 0: the same
//     scheme with the GEMM roles swapped (M = output channels, N = pixels), bit-identical results.
#include <atomic>
#include <stdio.h>
#include "conv_tc.cuh"
#include "sm90_ptx.cuh"

namespace lm {
namespace {

constexpr int BM = 128, BK = kBK, TILE_H = 16, TILE_W = 8;
constexpr int ROW_BYTES = 128;
constexpr int HALO_W = TILE_W + 2, HALO_H = TILE_H + 2;
constexpr int A_PLANE_BYTES_3x3 = HALO_W * HALO_H * ROW_BYTES;  // 180 rows x 128 B = 23040 B per plane
constexpr int A_PLANE_BYTES_1x1 = BM * ROW_BYTES;               // 16 KB per plane
constexpr int A_BUF_BYTES = 2 * A_PLANE_BYTES_3x3;              // 46080 B = 45 KB (both planes), 1024-aligned
constexpr int NUM_A_BUFS = 2;
constexpr int NUM_THREADS = 384;
constexpr int NUM_CONSUMER_WARPS = 8;
constexpr int MAX_CLASSES = 8;
constexpr int REGS_PRODUCER = 40, REGS_CONSUMER = 232;   // 128 x 40 + 256 x 232 <= 65536
// Split-plane output staging (fp16 build): one 64-channel half of a tile in the tile's last activation buffer, laid out
// as the store boxes (ConvMaps::out / pool, 128B-swizzled): 16 x 8 pixels x 2 planes, then the 8 x 4 pooled pixels.
constexpr int ST_PLANE = TILE_H * TILE_W * ROW_BYTES;                 // 16 KB
constexpr int ST_POOL = 2 * ST_PLANE;
constexpr int ST_POOL_PLANE = (TILE_H / 2) * (TILE_W / 2) * ROW_BYTES;  // 4 KB
static_assert(ST_POOL + 2 * ST_POOL_PLANE <= A_BUF_BYTES, "a tile's output half fits one activation buffer");

template <int BN>
struct Cfg {
  static constexpr int B_PLANE_BYTES = BN * ROW_BYTES;
  static constexpr int STAGE_BYTES = 2 * B_PLANE_BYTES;      // one weight tile (hi + lo planes) per k-block
  static constexpr int STAGES = (BN == 64) ? 6 : 4;
  // dynamic shared memory only (1024-aligned for the swizzled tiles): activation patches | weight ring | mbarriers | head
  // mbarriers: full / empty per weight stage, full / empty / staged per activation buffer, and the staging area's "free"
  static constexpr int NUM_BARS = 2 * STAGES + 3 * NUM_A_BUFS + 1;
  static constexpr int OFF_B = NUM_A_BUFS * A_BUF_BYTES;
  static constexpr int OFF_BARS = OFF_B + STAGES * STAGE_BYTES;
  static constexpr int OFF_HEAD = OFF_BARS + NUM_BARS * 8;                         // BN = 64 only: head weights + bias
  static constexpr int DYN_SMEM = OFF_HEAD + ((BN == 64) ? (MAX_CLASSES * 64 + MAX_CLASSES) * 4 : 0);
  static_assert(DYN_SMEM <= 232448, "shared-memory budget (227 KB per CTA)");
};

struct TileCoord {
  int n, y0, x0, n0;
};

__device__ __forceinline__ TileCoord decode_tile(int tile, int n_tiles, int tiles_x, int tiles_img, int BN) {
  TileCoord t;
  const int mt = tile / n_tiles;
  t.n0 = (tile - mt * n_tiles) * BN;
  t.n = mt / tiles_img;
  const int r = mt - t.n * tiles_img;
  const int ty = r / tiles_x;
  t.y0 = ty * TILE_H;
  t.x0 = (r - ty * tiles_x) * TILE_W;
  return t;
}

// The CTA's tiles.  MC = 1: every CTA on its own, tile = item.  MC = 2: the two CTAs of a cluster take two pixel tiles of
// the SAME output-channel block in lock step (work item = tile pair; every level has an even number of pixel tiles), so
// that they can share every weight stage.
template <int MC>
struct WorkItems {
  int first, step, total, n_tiles;
  uint32_t rank;
  __device__ WorkItems(int total_tiles, int n_tiles_) : n_tiles(n_tiles_) {
    rank = (MC > 1) ? cluster_ctarank() : 0u;
    first = (int)blockIdx.x / MC;
    step = (int)gridDim.x / MC;
    total = total_tiles / MC;
  }
  __device__ int tile(int item) const {
    if (MC == 1) return item;
    const int mtp = item / n_tiles;
    return (MC * mtp + (int)rank) * n_tiles + (item - mtp * n_tiles);
  }
};

#if !LM_OPERAND_F16
// the hi / lo operand planes of two adjacent channels (c even) of one pixel
__device__ __forceinline__ void store_split_pair(op_t* dst, size_t plane_stride, float a, float b) {
  float ha, la, hb, lb;
  split_tf32(a, ha, la);
  split_tf32(b, hb, lb);
  *reinterpret_cast<float2*>(dst) = make_float2(ha, hb);
  *reinterpret_cast<float2*>(dst + plane_stride) = make_float2(la, lb);
}
#endif

__device__ __forceinline__ float2 ldg2_or_zero(const float* p, int c) {
  return p ? __ldg(reinterpret_cast<const float2*>(p + c)) : make_float2(0.f, 0.f);
}

// Modes whose outputs are split planes that the consumers stage in shared memory and the storer warp writes with TMA.
__device__ __forceinline__ bool staged_stores(const ConvParams& p) {
  return LM_OPERAND_F16 && (p.mode == kModeReluBn || p.mode == kModeReluBnPool);
}

// One consumer warpgroup: the wgmma loop over every tile of the CTA for its 64 rows, then the tile's epilogue.
// The accumulator fragment of a thread covers two pixels - image rows y and y + 1 of column x - and BN / 4 channels
// (pairs c, c + 1 at c = n0 + 8 j + 2 (lane % 4)).
template <int BN, int TAPS, int MC>
__device__ __forceinline__ void conv_consumer(const ConvParams& p, uint32_t smem_a, uint32_t smem_b, uint32_t full0,
                                              uint32_t empty0, uint32_t afull0, uint32_t aempty0, uint32_t staged0,
                                              uint32_t sfree, const float* s_head_w, const float* s_head_b) {
  using C = Cfg<BN>;
  constexpr int NA = BN / 2;  // accumulator registers per thread for BN columns
  constexpr int STAGES = C::STAGES;
  constexpr int PATCH_W = (TAPS == 9) ? HALO_W : TILE_W;  // shared-memory rows per image row of the patch
  constexpr uint32_t A_PLANE = (uint32_t)((TAPS == 9) ? A_PLANE_BYTES_3x3 : A_PLANE_BYTES_1x1);
  constexpr uint32_t SBO_A = PATCH_W * ROW_BYTES;
  const int tid = threadIdx.x - 128;
  const int half = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int g = lane >> 2, qd = lane & 3;
  const int tiles_x = p.W / TILE_W, tiles_img = tiles_x * (p.H / TILE_H);
  const int n_tiles = p.Cout / BN;
  const int total_tiles = p.N * tiles_img * n_tiles;
  const int num_cb = (p.C0 + p.C1) / BK;
  const int num_kb = num_cb * TAPS, chunk_kb = p.chunk_kb;
  const uint32_t a_half = (uint32_t)(8 * half * PATCH_W * ROW_BYTES);
  const bool staged = staged_stores(p);   // the storer, not the consumers, frees each tile's last activation buffer

  const WorkItems<MC> items(total_tiles, n_tiles);
  float S[NA], P[NA], Q[NA];   // round-to-nearest sum of hi*hi | open chunk of hi*hi | corrections (x 2^11 for fp16)
  uint32_t s = 0, ph = 0, ab = 0, aph = 0;
  [[maybe_unused]] uint32_t fph = 0;   // parity of the staging area's "free" barrier (fp16 build)
  auto release = [&](uint32_t st, int a) {   // a weight stage (and an activation buffer, a >= 0) may be refilled
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(empty0 + 8 * st);
      if (MC > 1) mbar_arrive_cluster(empty0 + 8 * st, items.rank ^ 1u);   // the peer's producer also fills this stage
      if (a >= 0) mbar_arrive(aempty0 + 8 * a);
    }
  };
  auto mma_one = [&](float (&D)[NA], uint64_t da, uint64_t db, int acc) {
    if constexpr (BN == 128) wgmma_n128(D, da, db, acc); else wgmma_n64(D, da, db, acc);
  };

  for (int item = items.first; item < items.total; item += items.step) {
    const TileCoord t = decode_tile(items.tile(item), n_tiles, tiles_x, tiles_img, BN);
#pragma unroll
    for (int i = 0; i < NA; ++i) { S[i] = 0.f; Q[i] = 0.f; }
    // Chunks of chunk_kb k-blocks.  Inside a chunk every k-block is one committed wgmma group and the wait is for the
    // PREVIOUS group only, so the tensor core always has the next group queued; the chunk ends with an unconditional
    // wait for all groups before its hi*hi partial sum is read (every path to a read of P or Q passes a full wait, so
    // ptxas keeps the wgmmas asynchronous).
    for (int kb0 = 0; kb0 < num_kb; kb0 += chunk_kb) {
      const int kb1 = min(kb0 + chunk_kb, num_kb);
      uint32_t pend_s = 0;
      int pend_a = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        const int tap = (TAPS == 9) ? kb % 9 : 0;
        if (tap == 0) mbar_spin(afull0 + 8 * ab, aph);
        // tap (dy, dx) = the channel block's patch entered (dy * PATCH_W + dx) rows further
        const uint32_t a_tap = smem_a + ab * (uint32_t)A_BUF_BYTES + a_half + (uint32_t)(((tap / 3) * PATCH_W + (tap % 3)) * ROW_BYTES);
        const uint32_t b_st = smem_b + s * (uint32_t)C::STAGE_BYTES;
        mbar_spin(full0 + 8 * s, ph);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < ROW_BYTES / 32; ++k) {
          const uint64_t ah = make_desc_sw128(a_tap + 32 * k, SBO_A), al = make_desc_sw128(a_tap + A_PLANE + 32 * k, SBO_A);
          const uint64_t bh = make_desc_sw128(b_st + 32 * k, 1024), bl = make_desc_sw128(b_st + C::B_PLANE_BYTES + 32 * k, 1024);
          mma_one(P, ah, bh, k != 0 || kb != kb0);   // hi*hi (a chunk's first k-step restarts it from zero)
          mma_one(Q, ah, bl, 1);                      // hi*lo
          mma_one(Q, al, bh, 1);                      // lo*hi
        }
        wgmma_commit();
        if (kb > kb0) {
          wgmma_wait<1>();           // the previous k-block's group is done: its stage can be refilled
          release(pend_s, pend_a);
        }
        pend_s = s;
        // a channel block's last tap frees its activation buffer, except the tile's last one when it stages the outputs
        pend_a = (tap == TAPS - 1 && !(staged && kb == num_kb - 1)) ? (int)ab : -1;
        if (++s == STAGES) { s = 0; ph ^= 1u; }
        if (tap == TAPS - 1 && ++ab == NUM_A_BUFS) { ab = 0; aph ^= 1u; }
      }
      wgmma_wait<0>();
      release(pend_s, pend_a);
#pragma unroll
      for (int i = 0; i < NA; ++i) S[i] += P[i];
    }
#pragma unroll
    for (int i = 0; i < NA; ++i) S[i] += Q[i] * kLoUnscale;   // exact power-of-two rescale of hi*lo + lo*hi

    // ---- epilogue.  acc * in_unscale undoes the operands' power-of-two scales (1.0 unless the engine rescaled a
    // tensor); the product is exact, so fma(acc, unscale, bias) rounds exactly like the separate multiply and add.
    const float unscale = p.in_unscale;
    const int y = t.y0 + 8 * half + 2 * wq, x = t.x0 + g;   // registers 4j, 4j+1: row y; 4j+2, 4j+3: row y + 1
    const int c0 = t.n0 + 2 * qd;
    if (p.mode == kModeLinear) {
      float* out = static_cast<float*>(p.out);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = c0 + 8 * j;
        const float2 b = ldg2_or_zero(p.bias, c);
#pragma unroll
        for (int r = 0; r < 2; ++r)
          *reinterpret_cast<float2*>(out + (((size_t)t.n * p.H + y + r) * p.W + x) * p.Cout + c) =
              make_float2(__fmaf_rn(S[4 * j + 2 * r], unscale, b.x), __fmaf_rn(S[4 * j + 2 * r + 1], unscale, b.y));
      }
      continue;
    }
    // y = relu(acc + bias) * scale + shift   (Conv -> ReLU -> BatchNorm(eval), resunet.py:93-105).  The stored planes
    // hold y * out_scale: the power-of-two factor goes into scale and shift (it commutes with every rounding involved);
    // the head consumes y itself.
    const float cscale = (p.mode == kModeHead) ? 1.f : p.out_scale;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = c0 + 8 * j;
      const float2 b = ldg2_or_zero(p.bias, c), sc = ldg2_or_zero(p.scale, c), sh = ldg2_or_zero(p.shift, c);
      const float s0 = sc.x * cscale, s1 = sc.y * cscale, h0 = sh.x * cscale, h1 = sh.y * cscale;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float& v0 = S[4 * j + 2 * r];
        float& v1 = S[4 * j + 2 * r + 1];
        v0 = __fadd_rn(__fmul_rn(fmaxf(__fmaf_rn(v0, unscale, b.x), 0.f), s0), h0);
        v1 = __fadd_rn(__fmul_rn(fmaxf(__fmaf_rn(v1, unscale, b.y), 0.f), s1), h1);
      }
    }
    if (BN == 64 && p.mode == kModeHead) {
      // 1x1 head (resunet.py:69): the four lanes of a quad hold a pixel's 64 channels (16 each)
      float lg[2][MAX_CLASSES];
#pragma unroll
      for (int k = 0; k < MAX_CLASSES; ++k) {
        float d0 = 0.f, d1 = 0.f;
        if (k < p.K) {
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float w = s_head_w[k * 64 + 8 * j + 2 * qd + e];
              d0 = fmaf(w, S[4 * j + e], d0);
              d1 = fmaf(w, S[4 * j + 2 + e], d1);
            }
          }
        }
        d0 += __shfl_xor_sync(0xffffffffu, d0, 1);
        d1 += __shfl_xor_sync(0xffffffffu, d1, 1);
        d0 += __shfl_xor_sync(0xffffffffu, d0, 2);
        d1 += __shfl_xor_sync(0xffffffffu, d1, 2);
        lg[0][k] = (k < p.K) ? d0 + s_head_b[k] : -INFINITY;
        lg[1][k] = (k < p.K) ? d1 + s_head_b[k] : -INFINITY;
      }
      if (qd == 0) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float mx = -INFINITY;
#pragma unroll
          for (int k = 0; k < MAX_CLASSES; ++k) mx = fmaxf(mx, lg[r][k]);
          float se = 0.f;
#pragma unroll
          for (int k = 0; k < MAX_CLASSES; ++k) if (k < p.K) se += expf(lg[r][k] - mx);
          const float lse = logf(se);
          int best = 0;
          float bestv = -INFINITY;
#pragma unroll
          for (int k = 0; k < MAX_CLASSES; ++k) {
            if (k < p.K) {
              const float sc = (lg[r][k] - mx) - lse;  // LogSoftmax(dim=1), resunet.py:70
              if (sc > bestv) { bestv = sc; best = k; }  // first index wins ties (mask.py:185)
              if (p.scores) p.scores[(((size_t)t.n * p.K + k) * p.H + y + r) * p.W + x] = sc;
            }
          }
          p.labels[((size_t)t.n * p.H + y + r) * p.W + x] = (uint8_t)best;
        }
      }
      continue;
    }
#if LM_OPERAND_F16
    {  // fp16 saturates: report instead of storing inf (the engine lowers out_scale and runs again)
      bool ovf = false;
#pragma unroll
      for (int i = 0; i < NA; ++i) ovf |= !(fabsf(S[i]) <= kOpMax);
      if (__any_sync(0xffffffffu, ovf) && lane == 0 && p.range_flag) *p.range_flag = 1;
    }
    // Split planes (and their 2x2 average) staged in the tile's last activation buffer, one 64-channel half at a time, in
    // the layout of the store boxes: box row (x, y) holds 128 B of channels, its 16-byte chunk k at chunk k ^ (row % 8)
    // (128B swizzle).  The eight lanes of a chunk column hold eight consecutive box rows, so every store is conflict-free.
    // The storer warp hands each staged half to TMA.
    {
      const uint32_t buf = smem_a + (ab ^ 1u) * (uint32_t)A_BUF_BYTES;   // ab has moved past the tile's last channel block
      named_bar_sync(1, 256);   // both warpgroups' wgmmas have read the buffer (each reads halo rows of the other)
#pragma unroll
      for (int hc = 0; hc < BN / 64; ++hc) {
        if (hc > 0) {   // the storer's TMA has read the previous half
          mbar_spin(sfree, fph);
          fph ^= 1u;
        }
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = 8 * hc + jj;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            uint32_t hi, lo;
            split_f16x2(S[4 * j + 2 * r], S[4 * j + 2 * r + 1], hi, lo);
            const uint32_t row = (uint32_t)((8 * half + 2 * wq + r) * TILE_W + g);
            const uint32_t a = buf + row * ROW_BYTES + (uint32_t)(((jj ^ g) << 4) + 4 * qd);
            st_shared_u32(a, hi);
            st_shared_u32(a + ST_PLANE, lo);
          }
        }
        if (p.mode == kModeReluBnPool) {
          // 2x2 average (resunet.py:64): a thread holds rows y and y + 1 of column x, lane ^ 4 holds column x ^ 1;
          // (top-left + top-right) + (bottom-left + bottom-right), staged by the even-x lane
          const uint32_t prow = (uint32_t)((4 * half + wq) * (TILE_W / 2) + (g >> 1));
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = 8 * hc + jj;
            float pv[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float top = S[4 * j + e] + __shfl_xor_sync(0xffffffffu, S[4 * j + e], 4);
              const float bot = S[4 * j + 2 + e] + __shfl_xor_sync(0xffffffffu, S[4 * j + 2 + e], 4);
              pv[e] = (top + bot) * 0.25f;
            }
            if ((g & 1) == 0) {
              uint32_t hi, lo;
              split_f16x2(pv[0], pv[1], hi, lo);
              const uint32_t a = buf + ST_POOL + prow * ROW_BYTES + ((((uint32_t)jj ^ (prow & 7u)) << 4) + 4 * qd);
              st_shared_u32(a, hi);
              st_shared_u32(a + ST_POOL_PLANE, lo);
            }
          }
        }
        fence_proxy_async_smem();   // the staged half is visible to the TMA store that reads it
        __syncwarp();
        if (lane == 0) mbar_arrive(staged0 + 8 * (ab ^ 1u));
      }
    }
#else
    {
      const size_t plane = (size_t)p.H * p.W * p.Cout;
      op_t* img = static_cast<op_t*>(p.out) + (size_t)t.n * 2 * plane;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int r = 0; r < 2; ++r)
          store_split_pair(img + ((size_t)(y + r) * p.W + x) * p.Cout + c0 + 8 * j, plane, S[4 * j + 2 * r], S[4 * j + 2 * r + 1]);
    }
    if (p.mode == kModeReluBnPool) {
      // 2x2 average (resunet.py:64): a thread holds rows y and y + 1 of column x, lane ^ 4 holds column x ^ 1;
      // (top-left + top-right) + (bottom-left + bottom-right), stored by the even-x lane
      const int Hp = p.H / 2, Wp = p.W / 2;
      const size_t plane = (size_t)Hp * Wp * p.Cout;
      op_t* img = static_cast<op_t*>(p.out_pool) + (size_t)t.n * 2 * plane + ((size_t)(y >> 1) * Wp + (x >> 1)) * p.Cout + c0;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        float pv[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float top = S[4 * j + e] + __shfl_xor_sync(0xffffffffu, S[4 * j + e], 4);
          const float bot = S[4 * j + 2 + e] + __shfl_xor_sync(0xffffffffu, S[4 * j + 2 + e], 4);
          pv[e] = (top + bot) * 0.25f;
        }
        if ((g & 1) == 0) store_split_pair(img + 8 * j, plane, pv[0], pv[1]);
      }
    }
#endif
  }
}

// MC = 1: independent CTAs.  MC = 2 (weight multicast): clusters of two CTAs work on two pixel tiles of the same
// output-channel block in lock step; CTA r loads plane r (hi / lo) of every weight stage with one TMA multicast into both
// CTAs' rings, each CTA's full barrier counts the bytes of both loads, and a stage is free again when the consumers of BOTH
// CTAs have released it (empty barriers count the local and the remote arrivals).  Half the L2 -> SM weight bytes per MAC;
// activations, wgmmas and epilogue are per CTA and unchanged, so the results are bit-identical to MC = 1.
template <int BN, int MC>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
               const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmBX,
               const __grid_constant__ CUtensorMap tmOut, const __grid_constant__ CUtensorMap tmPool, const ConvParams p) {
  using C = Cfg<BN>;
  constexpr int STAGES = C::STAGES;
  extern __shared__ __align__(1024) uint8_t smem[];   // layout: Cfg<BN>; no static shared memory
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::OFF_BARS);
  float* s_head_w = reinterpret_cast<float*>(smem + C::OFF_HEAD);          // present for BN = 64 only (kModeHead)
  float* s_head_b = s_head_w + MAX_CLASSES * 64;
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = full0 + 8 * STAGES;
  const uint32_t afull0 = full0 + 16 * STAGES, aempty0 = afull0 + 8 * NUM_A_BUFS;
  const uint32_t staged0 = aempty0 + 8 * NUM_A_BUFS, sfree = staged0 + 8 * NUM_A_BUFS;
  const uint32_t smem_a = smem_u32(smem), smem_b = smem_a + C::OFF_B;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool staged = staged_stores(p);

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, MC * NUM_CONSUMER_WARPS); }
    for (int s = 0; s < NUM_A_BUFS; ++s) {
      mbar_init(afull0 + 8 * s, 1);
      mbar_init(aempty0 + 8 * s, NUM_CONSUMER_WARPS);
      mbar_init(staged0 + 8 * s, NUM_CONSUMER_WARPS);
    }
    mbar_init(sfree, 1);
    fence_mbar_init();
    tma_prefetch_desc(&tmA0); tma_prefetch_desc(&tmA1); tma_prefetch_desc(MC > 1 ? &tmBX : &tmB);
    if (staged) {
      tma_prefetch_desc(&tmOut);
      if (p.mode == kModeReluBnPool) tma_prefetch_desc(&tmPool);
    }
  }
  if (BN == 64 && p.mode == kModeHead) {
    for (int i = threadIdx.x; i < p.K * 64; i += NUM_THREADS) s_head_w[i] = p.head_w[i];
    if (threadIdx.x < p.K) s_head_b[threadIdx.x] = p.head_b[threadIdx.x];
  }
  __syncthreads();
  if (MC > 1) cluster_sync_all();   // the peer's barriers are initialised before any multicast load or remote arrive

  if (warp >= 4) {
    setmaxnreg_inc<REGS_CONSUMER>();
    if (p.taps == 9) conv_consumer<BN, 9, MC>(p, smem_a, smem_b, full0, empty0, afull0, aempty0, staged0, sfree, s_head_w, s_head_b);
    else conv_consumer<BN, 1, MC>(p, smem_a, smem_b, full0, empty0, afull0, aempty0, staged0, sfree, s_head_w, s_head_b);
  } else {
    setmaxnreg_dec<REGS_PRODUCER>();
    if (warp == 0) {
      // -------------------------------------------------------------- TMA producer (warp 0, one elected lane issues)
      const int tiles_x = p.W / TILE_W, tiles_img = tiles_x * (p.H / TILE_H);
      const int n_tiles = p.Cout / BN;
      const WorkItems<MC> items(p.N * tiles_img * n_tiles, n_tiles);
      const int taps = p.taps, halo = taps == 9 ? 1 : 0;
      const int num_cb = (p.C0 + p.C1) / BK;
      const uint32_t a_tx = 2u * (uint32_t)(taps == 9 ? A_PLANE_BYTES_3x3 : A_PLANE_BYTES_1x1);
      uint32_t s = 0, ph = 0, ab = 0, aph = 0;
      for (int item = items.first; item < items.total; item += items.step) {
        const TileCoord t = decode_tile(items.tile(item), n_tiles, tiles_x, tiles_img, BN);
        int c = 0;
        for (int cb = 0; cb < num_cb; ++cb, c += BK) {
          // the activation patch (+ halo) of this channel block, both planes, once for all taps
          mbar_wait_inline(aempty0 + 8 * ab, aph ^ 1);
          if (elect_one()) {
            mbar_arrive_expect_tx(afull0 + 8 * ab, a_tx);
            const uint32_t dst = smem_a + ab * A_BUF_BYTES;
            if (c < p.C0) tma_load_5d(dst, &tmA0, afull0 + 8 * ab, c, t.x0 - halo, t.y0 - halo, 0, t.n);
            else          tma_load_5d(dst, &tmA1, afull0 + 8 * ab, c - p.C0, t.x0 - halo, t.y0 - halo, 0, t.n);
          }
          __syncwarp();
          if (++ab == NUM_A_BUFS) { ab = 0; aph ^= 1; }
          for (int tap = 0; tap < taps; ++tap) {
            mbar_wait_inline(empty0 + 8 * s, ph ^ 1);
            if (elect_one()) {
              mbar_arrive_expect_tx(full0 + 8 * s, C::STAGE_BYTES);   // MC = 2: this CTA's plane and the peer's
              if (MC > 1)
                tma_load_4d_mcast(smem_b + s * C::STAGE_BYTES + items.rank * (uint32_t)C::B_PLANE_BYTES, &tmBX, full0 + 8 * s, c, t.n0,
                                  tap, (int)items.rank, (uint16_t)((1u << MC) - 1u));
              else
                tma_load_4d(smem_b + s * C::STAGE_BYTES, &tmB, full0 + 8 * s, c, t.n0, tap, 0);
            }
            __syncwarp();
            if (++s == STAGES) { s = 0; ph ^= 1; }
          }
        }
      }
    } else if (warp == 1 && staged) {
      // ------------------------------------------- storer (warp 1, lane 0 issues): the staged output halves to global
      const int tiles_x = p.W / TILE_W, tiles_img = tiles_x * (p.H / TILE_H);
      const int n_tiles = p.Cout / BN;
      const WorkItems<MC> items(p.N * tiles_img * n_tiles, n_tiles);
      const int num_cb = (p.C0 + p.C1) / BK;
      uint32_t nb = 0, sph = 0;   // activation buffers the producer has filled so far | staged parity, one bit per buffer
      for (int item = items.first; item < items.total; item += items.step) {
        const TileCoord t = decode_tile(items.tile(item), n_tiles, tiles_x, tiles_img, BN);
        const uint32_t b = (nb + (uint32_t)num_cb - 1u) % NUM_A_BUFS;   // the tile's last activation buffer
        nb += (uint32_t)num_cb;
#pragma unroll
        for (int hc = 0; hc < BN / 64; ++hc) {
          mbar_wait_inline(staged0 + 8 * b, (sph >> b) & 1u);
          sph ^= 1u << b;
          if (lane == 0) {
            const uint32_t src = smem_a + b * (uint32_t)A_BUF_BYTES;
            tma_store_5d(&tmOut, src, t.n0 + 64 * hc, t.x0, t.y0, 0, t.n);
            if (p.mode == kModeReluBnPool) tma_store_5d(&tmPool, src + ST_POOL, t.n0 + 64 * hc, t.x0 / 2, t.y0 / 2, 0, t.n);
            bulk_commit();
            bulk_wait_read<0>();
            if (hc + 1 < BN / 64) mbar_arrive(sfree);                       // the consumers may stage the next half
            else mbar_arrive_cnt(aempty0 + 8 * b, NUM_CONSUMER_WARPS);    // the producer may refill the buffer
          }
          __syncwarp();
        }
      }
      if (lane == 0) bulk_wait<0>();   // the outputs are in global memory before the CTA (and its cluster) finishes
    }
  }
  // MC = 2: no CTA leaves while its peer may still multicast into its shared memory or arrive on its barriers
  if (MC > 1) cluster_sync_all();
}

// ---------------------------------------------------------------------------------------------------------------------
// Channel-major tile for the 3x3 layers with 64 output channels (conv_cm64_fits), fp16-pair operands only.  The GEMM
// roles of conv_tc_kernel swapped:
//   * A operand = the weight stage, M = the 64 output channels (the BN = 64 kernel's weight box and descriptor).
//   * B operand = activations, N = 128 pixels per warpgroup.  A CTA takes 16 x 16 pixels of one image, warpgroup h the
//     columns 8h..8h+7 of all 16 rows, so that every 8-row group of the descriptor is one image row.  ONE 5-D TMA box per
//     64-channel block, (64 ch, 18 x, 18 y, 2 planes, 1 image) = 324 rows of 128 B per plane, serves all nine taps: tap
//     (dy, dx) of warpgroup h starts at row dy * 18 + dx + 8h with an 8-row-group stride of 18 rows.
//   * every wgmma is m64n128k16 (the BN = 64 kernel issues m64n64k16 with the same 4 KB of operands per instruction:
//     0.047 instead of 0.0625 B of shared-memory operand reads per MAC); per output pixel half the weight bytes and 1.27
//     instead of 1.41 input rows.
//   * the same three exact products per k-step, accumulated in the same order (hi*hi into P; act_hi*w_lo, then act_lo*w_hi
//     into Q), the same chunks and the same epilogue operations per element: the results equal the BN = 64 kernel's.
// Thread (warp w, g = lane / 4, qd = lane % 4) of warpgroup h holds in register 4j + e output channel 16w + g + 8 (e / 2)
// of pixel (row j, column 8h + 2qd + e % 2) of the tile.
constexpr int CM_TILE = 16, CM_HALO = CM_TILE + 2;
constexpr int CM_A_PLANE = CM_HALO * CM_HALO * ROW_BYTES;  // 324 rows x 128 B = 41472 B per plane
constexpr int CM_A_BUF = 2 * CM_A_PLANE;                   // 82944 B (both planes), 1024-aligned
constexpr int CM_STAGES = 3;
constexpr int CM_STAGE_BYTES = Cfg<64>::STAGE_BYTES;       // 16 KB: 64 cout x 64 cin, hi + lo planes
constexpr int CM_NUM_BARS = 2 * CM_STAGES + 3 * NUM_A_BUFS;   // full / empty per stage, full / empty / staged per buffer
constexpr int CM_OFF_B = NUM_A_BUFS * CM_A_BUF;
constexpr int CM_OFF_BARS = CM_OFF_B + CM_STAGES * CM_STAGE_BYTES;
constexpr int CM_OFF_HEAD = CM_OFF_BARS + CM_NUM_BARS * 8;
constexpr int CM_DYN_SMEM = CM_OFF_HEAD + (MAX_CLASSES * 64 + MAX_CLASSES) * 4;   // 217216 B
static_assert(CM_DYN_SMEM <= 232448, "shared-memory budget (227 KB per CTA)");
constexpr int CM_Y_STRIDE = 65;   // head: the tile's fp32 y staged [pixel][channel], padded against bank conflicts
static_assert(CM_TILE * CM_TILE * CM_Y_STRIDE * 4 <= CM_A_BUF, "the head's staging fits one activation buffer");
// split-plane staging: the tile's 16 x 16 pixels x 2 planes, then its 8 x 8 pooled pixels, as the store boxes lay them out
constexpr int CM_ST_PLANE = CM_TILE * CM_TILE * ROW_BYTES;                 // 32 KB
constexpr int CM_ST_POOL = 2 * CM_ST_PLANE;
constexpr int CM_ST_POOL_PLANE = (CM_TILE / 2) * (CM_TILE / 2) * ROW_BYTES;  // 8 KB
static_assert(CM_ST_POOL + 2 * CM_ST_POOL_PLANE <= CM_A_BUF, "a tile's outputs fit one activation buffer");

#if LM_OPERAND_F16
struct CmTile {
  int n, y0, x0;
};
__device__ __forceinline__ CmTile cm_tile(int tile, int tiles_x, int tiles_img) {
  CmTile t;
  t.n = tile / tiles_img;
  const int r = tile - t.n * tiles_img;
  const int ty = r / tiles_x;
  t.y0 = ty * CM_TILE;
  t.x0 = (r - ty * tiles_x) * CM_TILE;
  return t;
}

__device__ __forceinline__ void cm64_consumer(const ConvParams& p, uint8_t* smem, uint32_t smem_a, uint32_t smem_b,
                                              uint32_t full0, uint32_t empty0, uint32_t afull0, uint32_t aempty0,
                                              uint32_t staged0, const float* s_head_w, const float* s_head_b) {
  constexpr uint32_t SBO_X = CM_HALO * ROW_BYTES;
  const int tid = threadIdx.x - 128;
  const int half = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int g = lane >> 2, qd = lane & 3;
  const int tiles_x = p.W / CM_TILE, tiles_img = tiles_x * (p.H / CM_TILE);
  const int total_tiles = p.N * tiles_img;
  const int num_kb = (p.C0 + p.C1) / BK * 9, chunk_kb = p.chunk_kb;
  const bool head = p.mode == kModeHead;
  const uint32_t x_half = (uint32_t)(8 * half * ROW_BYTES);

  float S[64], P[64], Q[64];   // round-to-nearest sum of hi*hi | open chunk of hi*hi | corrections (x 2^11)
  uint32_t s = 0, ph = 0, ab = 0, aph = 0;
  auto release = [&](uint32_t st, int a) {   // a weight stage (and an activation buffer, a >= 0) may be refilled
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(empty0 + 8 * st);
      if (a >= 0) mbar_arrive(aempty0 + 8 * a);
    }
  };

  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const CmTile t = cm_tile(tile, tiles_x, tiles_img);
#pragma unroll
    for (int i = 0; i < 64; ++i) { S[i] = 0.f; Q[i] = 0.f; }
    // the k loop of conv_consumer (chunks, wait discipline, releases); the tile's last activation buffer stays taken until
    // the epilogue has staged y (head) or the outputs (the storer frees it) through it
    for (int kb0 = 0; kb0 < num_kb; kb0 += chunk_kb) {
      const int kb1 = min(kb0 + chunk_kb, num_kb);
      uint32_t pend_s = 0;
      int pend_a = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        const int tap = kb % 9;
        if (tap == 0) mbar_spin(afull0 + 8 * ab, aph);
        const uint32_t x_tap = smem_a + ab * (uint32_t)CM_A_BUF + x_half + (uint32_t)(((tap / 3) * CM_HALO + (tap % 3)) * ROW_BYTES);
        const uint32_t w_st = smem_b + s * (uint32_t)CM_STAGE_BYTES;
        mbar_spin(full0 + 8 * s, ph);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < ROW_BYTES / 32; ++k) {
          const uint64_t wh = make_desc_sw128(w_st + 32 * k, 1024), wl = make_desc_sw128(w_st + Cfg<64>::B_PLANE_BYTES + 32 * k, 1024);
          const uint64_t xh = make_desc_sw128(x_tap + 32 * k, SBO_X), xl = make_desc_sw128(x_tap + CM_A_PLANE + 32 * k, SBO_X);
          wgmma_n128(P, wh, xh, k != 0 || kb != kb0);   // hi*hi (a chunk's first k-step restarts it from zero)
          wgmma_n128(Q, wl, xh, 1);                      // act hi * w lo
          wgmma_n128(Q, wh, xl, 1);                      // act lo * w hi
        }
        wgmma_commit();
        if (kb > kb0) {
          wgmma_wait<1>();
          release(pend_s, pend_a);
        }
        pend_s = s;
        pend_a = (tap == 8 && kb != num_kb - 1) ? (int)ab : -1;
        if (++s == CM_STAGES) { s = 0; ph ^= 1u; }
        if (tap == 8 && ++ab == NUM_A_BUFS) { ab = 0; aph ^= 1u; }
      }
      wgmma_wait<0>();
      release(pend_s, pend_a);
#pragma unroll
      for (int i = 0; i < 64; ++i) S[i] += P[i];
    }
#pragma unroll
    for (int i = 0; i < 64; ++i) S[i] += Q[i] * kLoUnscale;

    // ---- epilogue: conv_consumer's operations per element, for the two channels c0 (e = 0, 1) and c0 + 8 (e = 2, 3)
    const float unscale = p.in_unscale;
    const float cscale = head ? 1.f : p.out_scale;
    const int c0 = 16 * wq + g;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int c = c0 + 8 * u;
      const float b = p.bias ? __ldg(p.bias + c) : 0.f;
      const float sc = (p.scale ? __ldg(p.scale + c) : 0.f) * cscale, sh = (p.shift ? __ldg(p.shift + c) : 0.f) * cscale;
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = S[4 * j + 2 * u + e];
          v = __fadd_rn(__fmul_rn(fmaxf(__fmaf_rn(v, unscale, b), 0.f), sc), sh);
        }
    }
    if (head) {
      // 1x1 head, log-softmax, argmax: one pixel per thread, from y staged in the tile's last activation buffer (the
      // wgmmas of both warpgroups have read it once both pass the first barrier).  The four partial sums over channels
      // 8j + 2q + e and their pairwise additions are those of conv_consumer's quad reduction.
      const int y_buf = (int)(ab ^ 1u);   // the buffer of the tile's last channel block
      float* ys = reinterpret_cast<float*>(smem + y_buf * CM_A_BUF);
      named_bar_sync(1, 256);
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          ys[(16 * j + 8 * half + 2 * qd + (e & 1)) * CM_Y_STRIDE + c0 + 8 * (e >> 1)] = S[4 * j + e];
      named_bar_sync(1, 256);
      const float* yp = ys + tid * CM_Y_STRIDE;
      float lg[MAX_CLASSES];
#pragma unroll
      for (int k = 0; k < MAX_CLASSES; ++k) {
        float d[4] = {0.f, 0.f, 0.f, 0.f};
        if (k < p.K) {
#pragma unroll
          for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) d[q] = fmaf(s_head_w[k * 64 + 8 * j + 2 * q + e], yp[8 * j + 2 * q + e], d[q]);
        }
        lg[k] = (k < p.K) ? ((d[0] + d[1]) + (d[2] + d[3])) + s_head_b[k] : -INFINITY;
      }
      fence_proxy_async_smem();   // the producer's next TMA load into this buffer comes after these accesses
      __syncwarp();
      if (lane == 0) mbar_arrive(aempty0 + 8 * y_buf);
      const int y = t.y0 + (tid >> 4), x = t.x0 + (tid & 15);
      float mx = -INFINITY;
#pragma unroll
      for (int k = 0; k < MAX_CLASSES; ++k) mx = fmaxf(mx, lg[k]);
      float se = 0.f;
#pragma unroll
      for (int k = 0; k < MAX_CLASSES; ++k) if (k < p.K) se += expf(lg[k] - mx);
      const float lse = logf(se);
      int best = 0;
      float bestv = -INFINITY;
#pragma unroll
      for (int k = 0; k < MAX_CLASSES; ++k) {
        if (k < p.K) {
          const float sc = (lg[k] - mx) - lse;  // LogSoftmax(dim=1), resunet.py:70
          if (sc > bestv) { bestv = sc; best = k; }  // first index wins ties (mask.py:185)
          if (p.scores) p.scores[(((size_t)t.n * p.K + k) * p.H + y) * p.W + x] = sc;
        }
      }
      p.labels[((size_t)t.n * p.H + y) * p.W + x] = (uint8_t)best;
      continue;
    }
    {  // fp16 saturates: report instead of storing inf (the engine lowers out_scale and runs again)
      bool ovf = false;
#pragma unroll
      for (int i = 0; i < 64; ++i) ovf |= !(fabsf(S[i]) <= kOpMax);
      if (__any_sync(0xffffffffu, ovf) && lane == 0 && p.range_flag) *p.range_flag = 1;
    }
    // Split planes, staged in the tile's last activation buffer in the layout of the store boxes (conv_consumer's:
    // 128-byte box rows of channels, 16-byte chunk k at chunk k ^ (row % 8)) for the storer warp's TMA stores.  Per image
    // row j and channel octet u the warp holds an 8 x 8 matrix (channel g, pixel column 2qd + e) in the movmatrix
    // fragment layout; its transpose gives lane (g, qd) channels 16w + 8u + 2qd, +1 of column 8h + g: the eight lanes of
    // a chunk column hold eight consecutive box rows.
    const uint32_t buf = smem_a + (ab ^ 1u) * (uint32_t)CM_A_BUF;   // ab has moved past the tile's last channel block
    named_bar_sync(1, 256);   // both warpgroups' wgmmas have read the buffer (each reads halo rows of the other)
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        uint32_t hi, lo;
        split_f16x2(S[4 * j + 2 * u], S[4 * j + 2 * u + 1], hi, lo);
        const uint32_t a = buf + (uint32_t)((16 * j + 8 * half + g) * ROW_BYTES + (((2 * wq + u) ^ g) << 4) + 4 * qd);
        st_shared_u32(a, movmatrix_trans(hi));
        st_shared_u32(a + CM_ST_PLANE, movmatrix_trans(lo));
      }
    if (p.mode == kModeReluBnPool) {
      // 2x2 average, ((top-left + top-right) + (bottom-left + bottom-right)) * 0.25, inside the thread: pooled pixel (row i,
      // column 4h + qd).  Pooled rows 2m and 2m + 1 pack into one matrix (channel g, column 2qd + r); after the transpose
      // lane (g, qd) holds channels 16w + 8u + 2qd, +1 of pooled pixel (row 2m + g % 2, column 4h + g / 2).
#pragma unroll
      for (int m = 0; m < 4; ++m)
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          float pv[2];
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int jt = 2 * (2 * m + r);
            const float top = S[4 * jt + 2 * u] + S[4 * jt + 2 * u + 1];
            const float bot = S[4 * (jt + 1) + 2 * u] + S[4 * (jt + 1) + 2 * u + 1];
            pv[r] = (top + bot) * 0.25f;
          }
          uint32_t hi, lo;
          split_f16x2(pv[0], pv[1], hi, lo);
          const int prow = (2 * m + (g & 1)) * (CM_TILE / 2) + 4 * half + (g >> 1);
          const uint32_t a = buf + CM_ST_POOL + (uint32_t)(prow * ROW_BYTES + (((2 * wq + u) ^ (prow & 7)) << 4) + 4 * qd);
          st_shared_u32(a, movmatrix_trans(hi));
          st_shared_u32(a + CM_ST_POOL_PLANE, movmatrix_trans(lo));
        }
    }
    fence_proxy_async_smem();   // the staged tile is visible to the TMA stores that read it
    __syncwarp();
    if (lane == 0) mbar_arrive(staged0 + 8 * (ab ^ 1u));
  }
}

// conv_tc_kernel's warp roles and mbarrier protocol (MC = 1) with the channel-major consumer; 3 weight stages.
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_cm64_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                 const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmOut,
                 const __grid_constant__ CUtensorMap tmPool, const ConvParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];   // activation buffers | weight ring | mbarriers | head
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + CM_OFF_BARS);
  float* s_head_w = reinterpret_cast<float*>(smem + CM_OFF_HEAD);
  float* s_head_b = s_head_w + MAX_CLASSES * 64;
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = full0 + 8 * CM_STAGES;
  const uint32_t afull0 = full0 + 16 * CM_STAGES, aempty0 = afull0 + 8 * NUM_A_BUFS, staged0 = aempty0 + 8 * NUM_A_BUFS;
  const uint32_t smem_a = smem_u32(smem), smem_b = smem_a + CM_OFF_B;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < CM_STAGES; ++s) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, NUM_CONSUMER_WARPS); }
    for (int s = 0; s < NUM_A_BUFS; ++s) {
      mbar_init(afull0 + 8 * s, 1);
      mbar_init(aempty0 + 8 * s, NUM_CONSUMER_WARPS);
      mbar_init(staged0 + 8 * s, NUM_CONSUMER_WARPS);
    }
    fence_mbar_init();
    tma_prefetch_desc(&tmA0); tma_prefetch_desc(&tmA1); tma_prefetch_desc(&tmB);
    if (p.mode != kModeHead) {
      tma_prefetch_desc(&tmOut);
      if (p.mode == kModeReluBnPool) tma_prefetch_desc(&tmPool);
    }
  }
  if (p.mode == kModeHead) {
    for (int i = threadIdx.x; i < p.K * 64; i += NUM_THREADS) s_head_w[i] = p.head_w[i];
    if (threadIdx.x < p.K) s_head_b[threadIdx.x] = p.head_b[threadIdx.x];
  }
  __syncthreads();

  if (warp >= 4) {
    setmaxnreg_inc<REGS_CONSUMER>();
    cm64_consumer(p, smem, smem_a, smem_b, full0, empty0, afull0, aempty0, staged0, s_head_w, s_head_b);
  } else {
    setmaxnreg_dec<REGS_PRODUCER>();
    if (warp == 0) {
      // -------------------------------------------------------------- TMA producer (warp 0, one elected lane issues)
      const int tiles_x = p.W / CM_TILE, tiles_img = tiles_x * (p.H / CM_TILE);
      const int num_cb = (p.C0 + p.C1) / BK;
      uint32_t s = 0, ph = 0, ab = 0, aph = 0;
      for (int tile = blockIdx.x; tile < p.N * tiles_img; tile += gridDim.x) {
        const CmTile t = cm_tile(tile, tiles_x, tiles_img);
        int c = 0;
        for (int cb = 0; cb < num_cb; ++cb, c += BK) {
          mbar_wait_inline(aempty0 + 8 * ab, aph ^ 1);
          if (elect_one()) {
            mbar_arrive_expect_tx(afull0 + 8 * ab, (uint32_t)CM_A_BUF);
            const uint32_t dst = smem_a + ab * CM_A_BUF;
            if (c < p.C0) tma_load_5d(dst, &tmA0, afull0 + 8 * ab, c, t.x0 - 1, t.y0 - 1, 0, t.n);
            else          tma_load_5d(dst, &tmA1, afull0 + 8 * ab, c - p.C0, t.x0 - 1, t.y0 - 1, 0, t.n);
          }
          __syncwarp();
          if (++ab == NUM_A_BUFS) { ab = 0; aph ^= 1; }
          for (int tap = 0; tap < 9; ++tap) {
            mbar_wait_inline(empty0 + 8 * s, ph ^ 1);
            if (elect_one()) {
              mbar_arrive_expect_tx(full0 + 8 * s, CM_STAGE_BYTES);
              tma_load_4d(smem_b + s * CM_STAGE_BYTES, &tmB, full0 + 8 * s, c, 0, tap, 0);
            }
            __syncwarp();
            if (++s == CM_STAGES) { s = 0; ph ^= 1; }
          }
        }
      }
    } else if (warp == 1 && p.mode != kModeHead) {
      // ------------------------------------------------- storer (warp 1, lane 0 issues): conv_tc_kernel's, one pass per tile
      const int tiles_x = p.W / CM_TILE, tiles_img = tiles_x * (p.H / CM_TILE);
      const int num_cb = (p.C0 + p.C1) / BK;
      uint32_t nb = 0, sph = 0;
      for (int tile = blockIdx.x; tile < p.N * tiles_img; tile += gridDim.x) {
        const CmTile t = cm_tile(tile, tiles_x, tiles_img);
        const uint32_t b = (nb + (uint32_t)num_cb - 1u) % NUM_A_BUFS;
        nb += (uint32_t)num_cb;
        mbar_wait_inline(staged0 + 8 * b, (sph >> b) & 1u);
        sph ^= 1u << b;
        if (lane == 0) {
          const uint32_t src = smem_a + b * (uint32_t)CM_A_BUF;
          tma_store_5d(&tmOut, src, 0, t.x0, t.y0, 0, t.n);
          if (p.mode == kModeReluBnPool) tma_store_5d(&tmPool, src + CM_ST_POOL, 0, t.x0 / 2, t.y0 / 2, 0, t.n);
          bulk_commit();
          bulk_wait_read<0>();
          mbar_arrive_cnt(aempty0 + 8 * b, NUM_CONSUMER_WARPS);
        }
        __syncwarp();
      }
      if (lane == 0) bulk_wait<0>();
    }
  }
}
#endif  // LM_OPERAND_F16

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) != cudaSuccess) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(f);
  }
  return fn;
}

#if LM_OPERAND_F16
constexpr CUtensorMapDataType kOpType = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
#else
constexpr CUtensorMapDataType kOpType = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
#endif

int encode(CUtensorMap* m, CUtensorMapDataType dtype, const void* base, int rank, const cuuint64_t* dims,
           const cuuint64_t* strides, const cuuint32_t* box) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return -1;
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(m, dtype, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box,
                  es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

// split-plane boxes of box_w x box_h pixels, BK channels, both planes, one image: activation loads (tile + halo) and
// output stores
int make_act_map(CUtensorMap* m, const void* base, int n_cap, int H, int W, int Cch, int box_w, int box_h) {
  const cuuint64_t E = kOpBytes;
  cuuint64_t dims[5] = {(cuuint64_t)Cch, (cuuint64_t)W, (cuuint64_t)H, 2, (cuuint64_t)n_cap};
  cuuint64_t strides[4] = {(cuuint64_t)Cch * E, (cuuint64_t)W * Cch * E, (cuuint64_t)H * W * Cch * E,
                           (cuuint64_t)2 * H * W * Cch * E};
  cuuint32_t box[5] = {BK, (cuuint32_t)box_w, (cuuint32_t)box_h, 2, 1};
  return encode(m, kOpType, base, 5, dims, strides, box);
}

}  // namespace

int make_conv_maps(ConvMaps* maps, const void* src0, const void* src1, const void* weights,
                   const ConvParams& p, int n_capacity) {
  const cuuint64_t E = kOpBytes;
  if (p.H % TILE_H || p.W % TILE_W || p.C0 % BK || p.C1 % BK || (p.taps != 1 && p.taps != 9)) return -2;
  const int BN = conv_tile_n(p);
  if (p.Cout % BN) return -3;
  const int halo = p.taps == 9 ? 2 : 0;
  // src1 absent: a1 repeats a0 (never read)
  const void* s1 = p.C1 > 0 ? src1 : src0;
  const int c1 = p.C1 > 0 ? p.C1 : p.C0;
  int r = make_act_map(&maps->a0, src0, n_capacity, p.H, p.W, p.C0, TILE_W + halo, TILE_H + halo);
  if (r) return r;
  r = make_act_map(&maps->a1, s1, n_capacity, p.H, p.W, c1, TILE_W + halo, TILE_H + halo);
  if (r) return r;
  if (conv_cm64_fits(p)) {
    r = make_act_map(&maps->a0cm, src0, n_capacity, p.H, p.W, p.C0, CM_HALO, CM_HALO);
    if (r) return r;
    r = make_act_map(&maps->a1cm, s1, n_capacity, p.H, p.W, c1, CM_HALO, CM_HALO);
    if (r) return r;
  }
#if LM_OPERAND_F16
  if (p.mode == kModeReluBn || p.mode == kModeReluBnPool) {
    const bool pool = p.mode == kModeReluBnPool, cm = conv_cm64_fits(p);
    const int Hp = p.H / 2, Wp = p.W / 2;
    r = make_act_map(&maps->out, p.out, n_capacity, p.H, p.W, p.Cout, TILE_W, TILE_H);
    if (!r && pool) r = make_act_map(&maps->pool, p.out_pool, n_capacity, Hp, Wp, p.Cout, TILE_W / 2, TILE_H / 2);
    if (!r && cm) r = make_act_map(&maps->outcm, p.out, n_capacity, p.H, p.W, p.Cout, CM_TILE, CM_TILE);
    if (!r && cm && pool) r = make_act_map(&maps->poolcm, p.out_pool, n_capacity, Hp, Wp, p.Cout, CM_TILE / 2, CM_TILE / 2);
    if (r) return r;
  }
#endif
  const int Cin = p.C0 + p.C1;
  cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)p.Cout, (cuuint64_t)p.taps, 2};
  cuuint64_t strides[3] = {(cuuint64_t)Cin * E, (cuuint64_t)p.Cout * Cin * E, (cuuint64_t)p.taps * p.Cout * Cin * E};
  cuuint32_t box[4] = {BK, (cuuint32_t)BN, 1, 2}, box_x[4] = {BK, (cuuint32_t)BN, 1, 1};   // both planes / one plane
  r = encode(&maps->b, kOpType, weights, 4, dims, strides, box);
  return r ? r : encode(&maps->bx, kOpType, weights, 4, dims, strides, box_x);
}


template <int BN, int MC>
static int launch_impl(const ConvMaps& maps, const ConvParams& p, int num_sms, cudaStream_t stream) {
  // the opt-in to > 48 KB of dynamic shared memory is a per-device function attribute
  static std::atomic<unsigned long long> attr_set_mask{0ull};  // engines of several host threads may launch concurrently
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return -9;
  if (!((attr_set_mask.load(std::memory_order_acquire) >> dev) & 1ull)) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<BN, MC>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::DYN_SMEM);
    if (e != cudaSuccess) return (int)e;
    attr_set_mask.fetch_or(1ull << dev, std::memory_order_release);
  }
  const int total = p.N * (p.H / TILE_H) * (p.W / TILE_W) * (p.Cout / BN);
  const int groups = total / MC, sm_groups = num_sms / MC;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(MC * (groups < sm_groups ? groups : sm_groups)), 1, 1);
  cfg.blockDim = dim3(NUM_THREADS, 1, 1);
  cfg.dynamicSmemBytes = Cfg<BN>::DYN_SMEM;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = MC; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, conv_tc_kernel<BN, MC>, maps.a0, maps.a1, maps.b, maps.bx, maps.out, maps.pool, p);
  return (int)(e != cudaSuccess ? e : cudaGetLastError());
}

// Sets the kernels' > 48 KB dynamic shared-memory opt-in on the current device (lm_create calls it, so that no launch -
// in particular none inside a CUDA-graph capture - has to).
int conv_tc_prepare() {
  cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<128, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<128>::DYN_SMEM);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_tc_kernel<64, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<64>::DYN_SMEM);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_tc_kernel<128, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<128>::DYN_SMEM);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_tc_kernel<64, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<64>::DYN_SMEM);
#if LM_OPERAND_F16
  if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_cm64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CM_DYN_SMEM);
#endif
  return (int)e;
}

int launch_conv_tc(const ConvMaps& maps, const ConvParams& p, int num_sms, cudaStream_t stream) {
  if (p.mode == kModeHead && (p.Cout != 64 || p.K > MAX_CLASSES)) return -4;
  if (p.chunk_kb < 1) return -5;
#if LM_OPERAND_F16
  if (p.conv64_cm && conv_cm64_fits(p)) {   // conv_tc_prepare has set the kernel's shared-memory opt-in
    const int total = p.N * (p.H / CM_TILE) * (p.W / CM_TILE);
    conv_cm64_kernel<<<total < num_sms ? total : num_sms, NUM_THREADS, CM_DYN_SMEM, stream>>>(maps.a0cm, maps.a1cm, maps.b, maps.outcm,
                                                                                          maps.poolcm, p);
    return (int)cudaGetLastError();
  }
#endif
  if (p.weight_mcast == 2)
    return conv_tile_n(p) == 128 ? launch_impl<128, 2>(maps, p, num_sms, stream) : launch_impl<64, 2>(maps, p, num_sms, stream);
  return conv_tile_n(p) == 128 ? launch_impl<128, 1>(maps, p, num_sms, stream) : launch_impl<64, 1>(maps, p, num_sms, stream);
}

}  // namespace lm
