// C-ABI engine (include/lungmask_b200.h): owns the device memory, the folded / split weights, the per-layer
// TMA descriptors and the kernel sequence that replaces LMInferer._inference (lungmask/mask.py:141-210).
#include <cuda.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>
#include <initializer_list>
#include <string>
#include <vector>

#include "../../include/lungmask_b200.h"
#include "conv_tc.cuh"
#include "forward_misc.cuh"
#include "postproc.cuh"
#include "preproc.cuh"
#include "shard.cuh"
#include "stats.cuh"
#include "clusters.cuh"
#include "regions.cuh"
#include "texture.cuh"
#include "shape.cuh"
#include "first_order.cuh"
#include "wavelet.cuh"
#include "filters.cuh"
#include "mesh.cuh"
#include "first_order_maps.cuh"
#include "glcm_maps.cuh"
#include "texture_maps.cuh"
#include "resample.cuh"
#include "laplacian.cuh"

using namespace lm;

namespace lm_impl {

thread_local std::string g_err;
thread_local unsigned g_fail_serial = 0;   // bumped by every fail(): RC() keeps a callee's own message instead of replacing it
int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  ++g_fail_serial;
  return code ? code : -1;
}
#define CU(x)                                                                                         \
  do {                                                                                                \
    cudaError_t e_ = (x);                                                                             \
    if (e_ != cudaSuccess) return fail((int)e_, "%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)
#define RC(x)                                                                            \
  do {                                                                                   \
    const unsigned serial_ = g_fail_serial;                                              \
    int r_ = (x);                                                                        \
    if (r_ && serial_ != g_fail_serial) return r_; /* the callee described the failure */ \
    if (r_) {                                                                            \
      const char* m_ = (r_ > 0 && r_ < 1000) ? cudaGetErrorString((cudaError_t)r_) : ""; \
      return fail(r_, "%s failed with code %d %s (%s:%d)", #x, r_, m_, __FILE__, __LINE__); \
    }                                                                                    \
  } while (0)

constexpr int R = LM_NET_RES;

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  int reserve(size_t want) {
    if (want <= n) return 0;
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
    cudaError_t e = cudaMalloc(&p, want * sizeof(T));
    if (e != cudaSuccess) return (int)e;
    n = want;
    return 0;
  }
  void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
};

// One convolution of the network in execution order.
struct LayerSpec {
  int level;      // spatial level: resolution 256 >> level
  int C0, C1, Cout, taps, mode;
  int src0, src1, dst, dst_pool;  // activation buffer ids (-1 = none)
};

// Activation buffers (ids).  "S" = split planes [N][2][H][W][C], "L" = single fp32 plane [N][H][W][C].
enum Act {
  A0, S0, P0, A1, S1, P1, A2, S2, P2, A3, S3, P3, A4, B4,  // encoder
  L0, U0, C0_, E0, L1, U1, C1_, E1, L2, U2, C2_, E2, L3, U3, C3_,  // decoder
  NUM_ACT
};
struct ActSpec { int level, C, split; };
const ActSpec ACT[NUM_ACT] = {
    {0, 64, 1}, {0, 64, 1}, {1, 64, 1}, {1, 128, 1}, {1, 128, 1}, {2, 128, 1}, {2, 256, 1}, {2, 256, 1}, {3, 256, 1},
    {3, 512, 1}, {3, 512, 1}, {4, 512, 1}, {4, 1024, 1}, {4, 1024, 1},
    {4, 512, 0}, {3, 512, 1}, {3, 512, 1}, {3, 512, 1}, {3, 256, 0}, {2, 256, 1}, {2, 256, 1}, {2, 256, 1},
    {2, 128, 0}, {1, 128, 1}, {1, 128, 1}, {1, 128, 1}, {1, 64, 0}, {0, 64, 1}, {0, 64, 1}};

constexpr int RANGE_STRIDE = NUM_ACT + 1;  // range flags per weight slot: one per activation tensor + one for the weights

// The 21 tensor-core convolutions (the stem 1->64 runs on CUDA cores). Order = execution order = blob order
// for the 3x3 layers (the four 1x1 "up" layers come after them in the blob, see lungmask_b200.h).
const LayerSpec LAYERS[] = {
    {0, 64, 0, 64, 9, kModeReluBnPool, A0, -1, S0, P0},      // down_path.0.block.3
    {1, 64, 0, 128, 9, kModeReluBn, P0, -1, A1, -1},         // down_path.1.block.0
    {1, 128, 0, 128, 9, kModeReluBnPool, A1, -1, S1, P1},    // down_path.1.block.3
    {2, 128, 0, 256, 9, kModeReluBn, P1, -1, A2, -1},        // down_path.2.block.0
    {2, 256, 0, 256, 9, kModeReluBnPool, A2, -1, S2, P2},    // down_path.2.block.3
    {3, 256, 0, 512, 9, kModeReluBn, P2, -1, A3, -1},        // down_path.3.block.0
    {3, 512, 0, 512, 9, kModeReluBnPool, A3, -1, S3, P3},    // down_path.3.block.3
    {4, 512, 0, 1024, 9, kModeReluBn, P3, -1, A4, -1},       // down_path.4.block.0
    {4, 1024, 0, 1024, 9, kModeReluBn, A4, -1, B4, -1},      // down_path.4.block.3
    {4, 1024, 0, 512, 1, kModeLinear, B4, -1, L0, -1},       // up_path.0.up.1 (below the upsample)
    {3, 512, 512, 512, 9, kModeReluBn, U0, S3, C0_, -1},     // up_path.0.conv_block.block.0  cat([up, bridge])
    {3, 512, 0, 512, 9, kModeReluBn, C0_, -1, E0, -1},       // up_path.0.conv_block.block.3
    {3, 512, 0, 256, 1, kModeLinear, E0, -1, L1, -1},        // up_path.1.up.1
    {2, 256, 256, 256, 9, kModeReluBn, U1, S2, C1_, -1},
    {2, 256, 0, 256, 9, kModeReluBn, C1_, -1, E1, -1},
    {2, 256, 0, 128, 1, kModeLinear, E1, -1, L2, -1},        // up_path.2.up.1
    {1, 128, 128, 128, 9, kModeReluBn, U2, S1, C2_, -1},
    {1, 128, 0, 128, 9, kModeReluBn, C2_, -1, E2, -1},
    {1, 128, 0, 64, 1, kModeLinear, E2, -1, L3, -1},         // up_path.3.up.1
    {0, 64, 64, 64, 9, kModeReluBn, U3, S0, C3_, -1},
    {0, 64, 0, 64, 9, kModeHead, C3_, -1, -1, -1},           // up_path.3.conv_block.block.3 + last + LogSoftmax + argmax
};
constexpr int NUM_LAYERS = sizeof(LAYERS) / sizeof(LAYERS[0]);
// upsample steps: after layer index -> (src L buffer, dst U buffer)
struct UpSpec { int after_layer, src, dst; };
const UpSpec UPS[4] = {{9, L0, U0}, {12, L1, U1}, {15, L2, U2}, {18, L3, U3}};

struct LayerWeights {
  float w_scale = 1.f;  // power of two: the planes hold w * w_scale, normalised to max |w * w_scale| in (2^14, 2^15]
  void* w = nullptr;  // op_t [2][taps][Cout][Cin] split
  float* bias = nullptr;
  float* scale = nullptr;
  float* shift = nullptr;
};
struct Slot {
  bool loaded = false;
  int K = 0;
  float *stem_w = nullptr, *stem_bias = nullptr, *stem_scale = nullptr, *stem_shift = nullptr;
  LayerWeights lw[NUM_LAYERS];
  float *head_w = nullptr, *head_b = nullptr;
  ConvMaps maps[NUM_LAYERS];
  ConvParams params[NUM_LAYERS];
  // Power-of-two scale of every split-plane activation tensor (conv_tc.cuh ConvParams::out_scale): all 1 until a value
  // of that tensor left fp16's range in some forward; then range_finish lowers the tensor's scale by 2^-8 (exactly
  // representable, no significand changes) and the forward runs again.  The state sticks to the weights it was found for.
  float act_scale[NUM_ACT];
  Slot() { for (float& s : act_scale) s = 1.f; }
};
// Tensors that feed one convolution together (virtual concat) or leave one epilogue together (block output + its
// pooled copy) share a scale: skip S_i, pooled P_i and the upsampled U_{3-i}.
int scale_group(int a) {
  switch (a) {
    case S0: case P0: case U3: return S0;
    case S1: case P1: case U2: return S1;
    case S2: case P2: case U1: return S2;
    case S3: case P3: case U0: return S3;
    default: return a;
  }
}

}  // namespace lm_impl
using namespace lm_impl;

struct lm_engine {
  int device = 0, B = 0, num_sms = 0;
  cudaStream_t st = nullptr;
  void* act[NUM_ACT] = {};  // split buffers: op_t planes; "L" buffers: fp32
  ShardView shard;             // multi-GPU slice sharding (lm_shard_*): gather blocks of all ranks
  bool shard_connected = false;
  int shard_test_slabs = 0;    // test hook (world == 1): label that many virtual slabs separately and join them
  int shard_slab_ccl = 1;      // 1: every rank labels its own slab, parents travel with the labels, boundaries are joined after
                               // the gather; 0: every rank labels the whole gathered volume
  uint32_t shard_epoch = 0;
  uint32_t* h_shard_err = nullptr;  // pinned copy of the block's error word
  int32_t* d_spare = nullptr;  // device int32[16]: spare label values computed on the device (fusion, mask.py:228)
  int* d_range = nullptr;   // device flags [LM_MAX_SLOTS][NUM_ACT + 1]: a value of activation tensor a (or, last entry, a
                            // weight) of that slot's network left the operand format's range (fp16 build: |x * scale| > 65504)
  int* h_range = nullptr;   // pinned host copy, refreshed at the end of every forward
  int range_slot = -1;      // the slot of the last forward (lm_debug_read_activation unscales with its scales)
  Slot slots[LM_MAX_SLOTS];
  // Whole-volume calls (run_volume): a host volume is uploaded to d_upload; volume_enqueue stages a volume that needs
  // re-orientation or conversion into d_vol / d_fvol, keeps the LPS mask in d_lps_out and the fusion's two masks in
  // d_native_l / d_native_r; a host call's results come back from d_out.
  DevBuf<uint8_t> d_upload;   // the host volume in its native orientation, raw bytes of any dtype
  DevBuf<int16_t> d_vol, d_resized;   // d_vol: the int16 LPS volume; also the upload of the stage taps and the sharded call
  DevBuf<uint8_t> d_fvol;     // the float32 / float64 LPS volume, raw bytes; also the upload of lm_preprocess_float
  DevBuf<uint8_t> d_lps_out, d_native_l, d_native_r;
  DevBuf<int32_t> d_boxes;
  // d_out: the mask of a host call, followed (lm_apply_volume_probs) by the (K, n0, n1, n2) probabilities at a 256-byte
  // aligned offset.  d_out and d_out2 are also the work buffers of the stage taps and d_out the sharded call's result.
  DevBuf<uint8_t> d_labels, d_post, d_out, d_out2, d_mask;
  DevBuf<float> d_scores, d_norm;   // d_scores: one wave of lm_forward's tap, or a whole volume of scores for the probabilities
  DevBuf<uint32_t> d_scratch;
  PostScratch post;
  LabelStatsWork stats;   // lm_label_stats_dev: counts, histograms and selection state
  ClusterWork clusters;   // lm_laa_clusters_dev: LAA maps, union-find parents, cluster sizes, size histogram
  RegionWork regions;     // lm_plane_label_counts_dev, lm_surface_distance_dev, lm_region_map_dev: EDT stacks, counts, LUT
  TextureWork texture;    // lm_texture_levels_dev, lm_glcm_dev, lm_glrlm_dev, lm_neighbour_counts_dev: error flag, counters
                          // (lm_zone_sizes_dev uses `clusters`)
  ShapeWork shape;        // lm_shape_sums_dev, lm_max_diameters_dev: sums, line tables, diameter candidates
  FirstOrderWork first_order;   // lm_first_order_sums_dev, lm_first_order_splits_dev: row table, histograms, sums
  WaveletWork wavelet;          // lm_wavelet_dev: the non-finite flag
  FilterWork filters;           // lm_image_range_dev, lm_image_filter_dev, lm_gradient_dev: a flag, the range partials
  MeshWork mesh;                // lm_mesh_counts_dev, lm_mesh_emit_dev: the triangle table, per-line counts and offsets
  FomWork fo_maps;              // lm_first_order_maps_dev: the error flag
  GlcmMapsWork glcm_maps;       // lm_glcm_maps_dev: the error flag
  TextureMapsWork texture_maps; // lm_texture_maps_dev: the error flag
  ResampleWork resample;        // lm_bspline_coefficients_dev, lm_resample_dev: the non-finite flag
  LogWork laplacian;            // lm_laplacian_of_gaussian_dev: the non-finite flag
  cudaEvent_t ev[8] = {};
  cudaEvent_t ev_conv[2] = {};
  std::vector<cudaEvent_t> ev_pool;  // per-launch event pairs when conv timing is on
  size_t ev_used = 0;
  bool time_convs = false;
  float last_conv_ms = 0.f;
  int64_t last_conv_launches = 0;
  cudaEvent_t ev_in = nullptr;       // lm_apply_dev: recorded on the caller's stream, waited for by the engine stream
  float last_ms[7] = {};
  int64_t launches = 0;
  // CUDA graphs of whole forwards (all waves of one volume: ~26 launches per wave), keyed by slot / buffers / slice count /
  // input type and valid for one configuration epoch (weights, options and activation scales bump it).  scores: the
  // volume-sized score buffer the head writes (lm_apply_volume_probs), nullptr for score-less forwards.
  struct FwdGraph { int slot; const void* in; uint8_t* labels; float* scores; int S; bool f32; uint64_t epoch; cudaGraphExec_t exec; int64_t launches; };
  std::vector<FwdGraph> graphs;
  uint64_t graph_epoch = 1;
  int use_graphs = 1;     // 0: launch every kernel individually (also whenever per-launch conv timing or score taps are on)
  int64_t graph_launches = 0, graph_hits = 0;
  unsigned bn64_mask = 0; // bit i: layer i of LAYERS uses BN = 64 output-channel tiles although Cout >= 128 (read at lm_load_weights)
  int stem_v2 = 3;        // stem kernel version: 0 stem_kernel, 1 stem_kernel_v2 - weights in registers, 4-pixel quads
                          // (bit-identical to stem_kernel, r02 GPU tests), 2 stem_kernel_v3 - shared input tile and weights,
                          // 3 (default) stem_kernel_v3 with the next tile's samples fetched one tile ahead
  int upsample_v2 = 2;    // 2 (default): upsample2x_cells_kernel<true> - one load per output sample, corners indexed statically;
                          // 1: the same with run-time corner selection, 0: upsample2x_kernel (all three bit-identical)
  int weight_mcast = 0;   // 2: clusters of two CTAs share each weight stage through TMA multicast (conv_tc.cu, MC = 2)
  int chunk_kb = 1;       // k-blocks per tensor-core chunk of hi*hi (conv_tc.cu) for the 64-channel layers
  int chunk_kb_wide = 2;  // ... for the layers with Cout >= 128
  int conv64_cm = 1;      // 1: the 3x3 layers with 64 output channels run conv_cm64_kernel; 0: the BN = 64 kernel (bit-identical)
};

namespace {

size_t blob_floats(int K) {
  size_t n = 0;
  // 18 conv3x3 (+BN): stem + the 3x3 entries of LAYERS
  n += 64 * 1 * 9 + 64 * 5;
  for (int i = 0; i < NUM_LAYERS; ++i)
    if (LAYERS[i].taps == 9) n += (size_t)LAYERS[i].Cout * (LAYERS[i].C0 + LAYERS[i].C1) * 9 + (size_t)LAYERS[i].Cout * 5;
  for (int i = 0; i < NUM_LAYERS; ++i)
    if (LAYERS[i].taps == 1) n += (size_t)LAYERS[i].Cout * LAYERS[i].C0 + LAYERS[i].Cout;
  n += (size_t)K * 64 + K;
  return n;
}

// BatchNorm2d(eval) as torch evaluates it on CPU: invstd = 1/sqrt(var+eps); alpha = invstd*gamma; beta = b - mean*alpha
void fold_bn(const float* g, const float* b, const float* mean, const float* var, int C, std::vector<float>& scale,
             std::vector<float>& shift) {
  scale.resize(C);
  shift.resize(C);
  for (int c = 0; c < C; ++c) {
    const float invstd = 1.0f / sqrtf(var[c] + 1e-5f);
    const float alpha = invstd * g[c];
    scale[c] = alpha;
    shift[c] = b[c] - mean[c] * alpha;
  }
}

// Stream-ordered upload: every consumer runs on the engine stream (which does not synchronise with the
// legacy default stream), and a pageable cudaMemcpy may return before its DMA has landed.
int upload(float** dst, const float* src, size_t n, cudaStream_t st) {
  if (*dst == nullptr) {
    cudaError_t e = cudaMalloc(dst, n * sizeof(float));
    if (e != cudaSuccess) return (int)e;
  }
  cudaError_t e = cudaMemcpyAsync(*dst, src, n * sizeof(float), cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return (int)e;
  return (int)cudaStreamSynchronize(st);
}

// d_in: the resized slices, int16 HU (in_f32 == false) or the normalised fp32 network input of a float volume
int forward_batch(lm_engine* e, Slot& s, const void* d_in, bool in_f32, int n, uint8_t* d_labels, float* d_scores,
                  bool time_convs) {
  int* const range = e->d_range + (size_t)(&s - e->slots) * RANGE_STRIDE;
  if (in_f32)
    RC(launch_stem_f32(static_cast<const float*>(d_in), e->act[A0], s.stem_w, s.stem_bias, s.stem_scale, s.stem_shift, n, R, R,
                       range + A0, s.act_scale[A0], e->stem_v2, e->num_sms, e->st));
  else
    RC(launch_stem_any(static_cast<const int16_t*>(d_in), e->act[A0], s.stem_w, s.stem_bias, s.stem_scale, s.stem_shift, n, R, R,
                       range + A0, s.act_scale[A0], e->stem_v2, e->num_sms, e->st));
  e->launches++;
  int up = 0;
  for (int i = 0; i < NUM_LAYERS; ++i) {
    ConvParams p = s.params[i];
    p.N = n;
    p.chunk_kb = (p.Cout >= 128) ? e->chunk_kb_wide : e->chunk_kb;
    p.weight_mcast = e->weight_mcast;
    p.conv64_cm = e->conv64_cm;
    const LayerSpec& L = LAYERS[i];
    p.range_flag = L.dst >= 0 ? range + L.dst : nullptr;
    p.in_unscale = 1.f / (s.act_scale[L.src0] * s.lw[i].w_scale);   // src1 (virtual concat) shares src0's scale group
    p.out_scale = (L.mode == kModeReluBn || L.mode == kModeReluBnPool) ? s.act_scale[L.dst] : 1.f;
    if (p.mode == kModeHead) { p.labels = d_labels; p.scores = d_scores; }
    if (time_convs) {
      if (e->ev_used + 2 > e->ev_pool.size()) {
        for (int k = 0; k < 64; ++k) { cudaEvent_t ev; CU(cudaEventCreate(&ev)); e->ev_pool.push_back(ev); }
      }
      cudaEventRecord(e->ev_pool[e->ev_used], e->st);
    }
    RC(launch_conv_tc(s.maps[i], p, e->num_sms, e->st));
    if (time_convs) { cudaEventRecord(e->ev_pool[e->ev_used + 1], e->st); e->ev_used += 2; }
    e->launches++;
    if (up < 4 && UPS[up].after_layer == i) {
      const ActSpec& src = ACT[UPS[up].src];
      RC((e->upsample_v2 >= 2 ? launch_upsample2x_cells_static : e->upsample_v2 ? launch_upsample2x_cells : launch_upsample2x)(
          static_cast<const float*>(e->act[UPS[up].src]), e->act[UPS[up].dst], n,
                                                                      R >> src.level, R >> src.level, src.C, range + UPS[up].dst,
                                                                      s.act_scale[UPS[up].dst], e->num_sms, e->st));
      e->launches++;
      ++up;
    }
  }
  return 0;
}

int drain_conv_events(lm_engine* e) {
  float total = 0.f;
  for (size_t i = 0; i + 1 < e->ev_used; i += 2) {
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, e->ev_pool[i], e->ev_pool[i + 1]));
    total += ms;
  }
  e->last_conv_ms = total;
  e->last_conv_launches = (int64_t)(e->ev_used / 2);
  e->ev_used = 0;
  return 0;
}

void drop_graphs(lm_engine* e) {
  for (auto& g : e->graphs) cudaGraphExecDestroy(g.exec);
  e->graphs.clear();
}

// Replays (or first captures) the kernel sequence of one volume's forward - every wave's stem, 21 tensor-core
// convolutions and 4 upsamples - as ONE graph launch on the engine stream.  Returns 0 when the graph was launched,
// 1 when graphs cannot be used (the caller launches the kernels one by one), < 0 on a real error.
// d_vol_scores: nullptr, or the (S, K, 256, 256) buffer the head writes every slice's log-softmax scores to.
int forward_graph(lm_engine* e, int slot, const void* d_in, int S, uint8_t* d_labels, bool in_f32, float* d_vol_scores) {
  Slot& s = e->slots[slot];
  for (auto& g : e->graphs) {
    if (g.slot == slot && g.in == d_in && g.labels == d_labels && g.scores == d_vol_scores && g.S == S && g.f32 == in_f32 &&
        g.epoch == e->graph_epoch) {
      CU(cudaGraphLaunch(g.exec, e->st));
      e->launches += g.launches;
      e->graph_hits++;
      return 0;
    }
  }
  if (e->graphs.size() >= 24 || (!e->graphs.empty() && e->graphs[0].epoch != e->graph_epoch)) drop_graphs(e);
  if (cudaStreamBeginCapture(e->st, cudaStreamCaptureModeRelaxed) != cudaSuccess) { cudaGetLastError(); e->use_graphs = 0; return 1; }
  const int64_t before = e->launches;
  int rc = 0;
  for (int s0 = 0; s0 < S && rc == 0; s0 += e->B) {
    const int n = S - s0 < e->B ? S - s0 : e->B;
    const void* in_wave = in_f32 ? static_cast<const void*>(static_cast<const float*>(d_in) + (size_t)s0 * R * R)
                                 : static_cast<const void*>(static_cast<const int16_t*>(d_in) + (size_t)s0 * R * R);
    rc = forward_batch(e, s, in_wave, in_f32, n, d_labels + (size_t)s0 * R * R,
                       d_vol_scores ? d_vol_scores + (size_t)s0 * s.K * R * R : nullptr, false);
  }
  cudaGraph_t graph = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(e->st, &graph);
  const int64_t captured = e->launches - before;
  e->launches = before;
  if (rc != 0 || ce != cudaSuccess || !graph) {
    if (graph) cudaGraphDestroy(graph);
    cudaGetLastError();
    e->use_graphs = 0;   // stay on plain launches for the rest of this engine's life
    return rc < 0 ? rc : 1;
  }
  cudaGraphExec_t exec = nullptr;
  const cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ie != cudaSuccess || !exec) { cudaGetLastError(); e->use_graphs = 0; return 1; }
  e->graphs.push_back({slot, d_in, d_labels, d_vol_scores, S, in_f32, e->graph_epoch, exec, captured});
  CU(cudaGraphLaunch(exec, e->st));
  e->launches += captured;
  e->graph_launches++;
  return 0;
}

// h_scores: the parity tap (host, synchronised per wave, plain launches).  d_vol_scores: a device buffer of the whole
// volume's scores (S, K, 256, 256); each wave's head writes its slices at offset s0 * K * 256 * 256, graph-captured.
int forward_all(lm_engine* e, int slot, const void* d_in, int S, uint8_t* d_labels, float* h_scores,
                float* conv_ms, bool in_f32 = false, float* d_vol_scores = nullptr) {
  if (slot < 0 || slot >= LM_MAX_SLOTS || !e->slots[slot].loaded) return fail(-30, "weight slot %d not loaded", slot);
  Slot& s = e->slots[slot];
  float* d_scores = nullptr;
  if (h_scores) {
    RC(e->d_scores.reserve((size_t)e->B * s.K * R * R));
    d_scores = e->d_scores.p;
  }
  const bool timing = conv_ms != nullptr || e->time_convs;
  if (e->use_graphs && !timing && !h_scores) {
    int gr = forward_graph(e, slot, d_in, S, d_labels, in_f32, d_vol_scores);
    if (gr == 0) {
      CU(cudaMemcpyAsync(e->h_range, e->d_range, LM_MAX_SLOTS * RANGE_STRIDE * sizeof(int), cudaMemcpyDeviceToHost, e->st));
      e->range_slot = slot;
      return 0;
    }
    if (gr < 0) return gr;   // gr > 0: graphs are unavailable here (capture failed) - fall through to plain launches
  }
  for (int s0 = 0; s0 < S; s0 += e->B) {
    const int n = S - s0 < e->B ? S - s0 : e->B;
    const void* in_wave = in_f32 ? static_cast<const void*>(static_cast<const float*>(d_in) + (size_t)s0 * R * R)
                                 : static_cast<const void*>(static_cast<const int16_t*>(d_in) + (size_t)s0 * R * R);
    float* const wave_scores = d_vol_scores ? d_vol_scores + (size_t)s0 * s.K * R * R : d_scores;
    RC(forward_batch(e, s, in_wave, in_f32, n, d_labels + (size_t)s0 * R * R, wave_scores, conv_ms != nullptr || e->time_convs));
    if (h_scores) {
      CU(cudaMemcpyAsync(h_scores + (size_t)s0 * s.K * R * R, d_scores, (size_t)n * s.K * R * R * sizeof(float),
                         cudaMemcpyDeviceToHost, e->st));
      CU(cudaStreamSynchronize(e->st));
    }
  }
  CU(cudaMemcpyAsync(e->h_range, e->d_range, LM_MAX_SLOTS * RANGE_STRIDE * sizeof(int), cudaMemcpyDeviceToHost, e->st));  // read by range_finish after the caller's sync
  e->range_slot = slot;
  if (conv_ms) {  // device time of the tensor-core convolution launches alone (CUDA events on the launch stream)
    CU(cudaStreamSynchronize(e->st));
    RC(drain_conv_events(e));
    *conv_ms = e->last_conv_ms;
  }
  return 0;
}

// Probability output of inference_dev (lm_apply_volume_probs): the head writes the volume's scores to `scores`
// (S, K, 256, 256), and after the mask reshape probs_device writes (K, n0, n1, n2) to `probs` in the native orientation
// given by perm / flip (identity: the volume is LPS).
struct ProbOut { float* scores; float* probs; int perm[3]; int flip[3]; };

// ev[1]; bodymask + resize of S slices (S, H, W) into the network input d_resized / d_norm; ev[2]; the forward; ev[3].
// vtype: 0 = int16 HU volume, 1 = float32, 2 = float64 (float volumes keep their dtype through the reference's
// pre-processing and normalisation; preproc.cu resize_kernel).  boxes (S, 4), labels (S, 256, 256) and scores (nullptr,
// or (S, K, 256, 256)) are the caller's.  S == 0 (a rank without slices): the events alone.
int forward_head(lm_engine* e, int slot, const void* d_vol, int vtype, int S, int H, int W, int32_t* boxes, uint8_t* labels,
                 float* scores) {
  const size_t nr = (size_t)S * R * R;
  if (S > 0) RC(vtype == 0 ? e->d_resized.reserve(nr) : e->d_norm.reserve(nr));
  CU(cudaEventRecord(e->ev[1], e->st));
  if (S > 0) {
    if (vtype == 0) {
      RC(launch_bodymask(static_cast<const int16_t*>(d_vol), S, H, W, boxes, nullptr, e->num_sms, e->st));
      RC(launch_resize(static_cast<const int16_t*>(d_vol), S, H, W, boxes, e->d_resized.p, R, R, 1, e->num_sms, e->st));
    } else {
      RC(launch_bodymask_float(d_vol, vtype == 2, S, H, W, boxes, nullptr, e->num_sms, e->st));
      RC(launch_resize_float(d_vol, vtype == 2, S, H, W, boxes, e->d_norm.p, R, R, e->num_sms, e->st));
    }
    e->launches += 2;
  }
  CU(cudaEventRecord(e->ev[2], e->st));
  if (S > 0) {
    const void* net_in = vtype == 0 ? static_cast<const void*>(e->d_resized.p) : e->d_norm.p;
    RC(forward_all(e, slot, net_in, S, labels, nullptr, nullptr, vtype != 0, scores));
  }
  CU(cudaEventRecord(e->ev[3], e->st));
  return 0;
}

// preprocess -> forward -> postprocess -> reshape of an LPS volume, all device-resident. d_out: (S,H,W) uint8.
int inference_dev(lm_engine* e, int slot, const void* d_vol, int vtype, int S, int H, int W, int flags, uint8_t* d_out,
                  const ProbOut* prob) {
  const size_t nr = (size_t)S * R * R;
  RC(e->d_boxes.reserve((size_t)S * 4));
  RC(e->d_labels.reserve(nr));
  RC(e->d_post.reserve(nr));
  RC(forward_head(e, slot, d_vol, vtype, S, H, W, e->d_boxes.p, e->d_labels.p, prob ? prob->scores : nullptr));
  const uint8_t* masks = e->d_labels.p;
  if (!(flags & LM_FLAG_NO_POSTPROCESS)) {
    // labels out of the argmax are < K: the post-processing needs no host round trip to learn which occur
    RC(postprocess_device(e->post, e->d_labels.p, S, R, R, nullptr, 0, nullptr, 0, 3, e->slots[slot].K - 1, e->d_post.p, e->num_sms,
                          e->st, &e->launches));
    masks = e->d_post.p;
  }
  CU(cudaEventRecord(e->ev[4], e->st));
  RC(reshape_device(masks, e->d_boxes.p, S, H, W, R, R, d_out, e->num_sms, e->st));
  e->launches++;
  if (prob) {
    const int dl[3] = {S, H, W};
    RC(probs_device(prob->scores, e->d_boxes.p, e->slots[slot].K, R, R, dl, prob->perm, prob->flip, prob->probs, e->num_sms, e->st));
    e->launches++;
  }
  CU(cudaEventRecord(e->ev[5], e->st));
  return 0;
}

// The lowest scale of a group: 4 steps of 2^-8, for values up to 65504 * 2^32 = 2.8e14.
constexpr float kMinActScale = 0x1p-32f;

// After a stream synchronisation: did any activation leave the operand format's range during the forward passes?
// Returns 0 (no), 1 (yes: the offending groups' power-of-two scales were lowered - run the forward again) or an error.
// A flag counts only when no tensor upstream of it flagged in the same forward.  An overflowing tensor is stored as
// +inf / -inf planes: behind a ReLU its consumers see 0 instead of NaN, behind a 1x1 layer (no ReLU) NaN reaches the
// upsample, which flags it - either way every tensor downstream holds wrong values, and lowering their groups would
// only cost them precision.  The first flag of a cascade is always genuine (its inputs were in range), so every re-run
// lowers at least one group; a group that would go below kMinActScale ends the call with LM_ERR_RANGE.
int range_finish(lm_engine* e) {
  bool any = false;
  for (int i = 0; i < LM_MAX_SLOTS * RANGE_STRIDE; ++i) any |= e->h_range[i] != 0;
  if (!any) return 0;
  cudaMemsetAsync(e->d_range, 0, LM_MAX_SLOTS * RANGE_STRIDE * sizeof(int), e->st);
  bool weight_flag = false, give_up = false;
  bool lower[LM_MAX_SLOTS][NUM_ACT] = {};   // [slot][group representative]: one step of 2^-8 this re-run
  for (int sl = 0; sl < LM_MAX_SLOTS; ++sl) {
    int* h = e->h_range + sl * RANGE_STRIDE;
    weight_flag |= h[NUM_ACT] != 0;
    bool tainted[NUM_ACT] = {};   // a tensor upstream of this one flagged (execution order visits sources first)
    auto feed = [&](int src, int dst) { if (src >= 0 && dst >= 0 && (h[src] || tainted[src])) tainted[dst] = true; };
    for (int i = 0, up = 0; i < NUM_LAYERS; ++i) {
      const LayerSpec& L = LAYERS[i];
      for (int d : {L.dst, L.dst_pool}) { feed(L.src0, d); feed(L.src1, d); }
      if (up < 4 && UPS[up].after_layer == i) { feed(UPS[up].src, UPS[up].dst); ++up; }
    }
    for (int a = 0; a < NUM_ACT; ++a) {
      if (!h[a] || tainted[a]) continue;
      const int g = scale_group(a);
      lower[sl][g] = true;
      give_up |= e->slots[sl].act_scale[g] <= kMinActScale;
    }
    for (int i = 0; i < RANGE_STRIDE; ++i) h[i] = 0;
  }
  if (weight_flag || give_up)
    return fail(LM_ERR_RANGE, "an activation exceeded the fp16 operand range even after rescaling by 2^-32 (|x| > 2.8e14): "
                              "the weights are not a usable network (rebuild with -DLM_OPERAND_F16=0 for tf32 operands)");
  for (int sl = 0; sl < LM_MAX_SLOTS; ++sl)
    for (int b = 0; b < NUM_ACT; ++b)   // one step per group and re-run, whichever members raised their flags
      if (lower[sl][scale_group(b)]) e->slots[sl].act_scale[b] *= (1.f / 256.f);
  e->graph_epoch++;
  return 1;
}

// Enqueue-synchronise-verify: `enqueue` puts a whole call on the engine stream; after the synchronisation the
// post-processing reports whether its region tables were large enough (the region count lives on the device).  If not,
// the tables grow to the reported size and the call is enqueued once more (a label map with more than one region per 32
// voxels; never seen with a trained network).  range_finish lowers at least one group's scale per re-run and at most
// 4 times per group, so range rescues end on their own after fewer than 4 * NUM_ACT re-runs.
template <typename F>
int run_checked(lm_engine* e, F&& enqueue) {
  for (int attempt = 0;; ++attempt) {
    RC(enqueue());
    CU(cudaStreamSynchronize(e->st));
    const int rr = range_finish(e);   // 1: a tensor left fp16's range, its scale was lowered -> run again (exact rescale)
    if (rr < 0) return rr;
    const int pf = postprocess_finish(e->post);
    if (!rr && !pf) return 0;
    if (attempt >= 8 + 4 * NUM_ACT) return fail(-22, "the call did not settle after %d re-runs (region tables %u regions / operand range)", attempt, e->post.last_regions);
    if (pf) RC(e->post.reserve_regions(e->post.want_regions));
  }
}

void shard_release(lm_engine* e) {
  for (int p = 0; p < e->shard.world; ++p) {
    if (!e->shard.block[p]) continue;
    if (p == e->shard.rank) cudaFree(e->shard.block[p]); else cudaIpcCloseMemHandle(e->shard.block[p]);
    e->shard.block[p] = nullptr;
  }
  if (e->h_shard_err) cudaFreeHost(e->h_shard_err);
  e->h_shard_err = nullptr;
  e->shard = ShardView();
  e->shard_connected = false;
}

void shard_range(int S, int rank, int world, int* lo, int* hi) {
  const int per = (S + world - 1) / world;
  *lo = rank * per < S ? rank * per : S;
  *hi = *lo + per < S ? *lo + per : S;
}

// One volume, slices sharded over the ranks: per-slice stages on this rank's slab, results written straight into the
// rank's gather block, pushed to the peers, post-processing + reshape replicated on the gathered volume (SURVEY 8e).
// d_vol / d_out: WHOLE volume on this rank's device (only the slab of d_vol is read).
int sharded_dev(lm_engine* e, int slot, const int16_t* d_vol, int S, int H, int W, int flags, uint8_t* d_out) {
  const ShardView& v = e->shard;
  if (slot < 0 || slot >= LM_MAX_SLOTS || !e->slots[slot].loaded) return fail(-30, "weight slot %d not loaded", slot);
  int lo, hi;
  shard_range(S, v.rank, v.world, &lo, &hi);
  const size_t plane = (size_t)H * W, rr = (size_t)R * R;
  uint8_t* labels_full = v.block[v.rank] + shard_labels_offset(v.slice_cap);
  int32_t* boxes_full = reinterpret_cast<int32_t*>(v.block[v.rank] + shard_boxes_offset());
  const uint32_t epoch = ++e->shard_epoch;
  const int ns = hi - lo;
  RC(forward_head(e, slot, d_vol + (size_t)lo * plane, 0, ns, H, W, boxes_full + 4 * (size_t)lo, labels_full + (size_t)lo * rr,
                  nullptr));
  // slab-sharded 3-D labelling (SURVEY 8f-1): this rank labels its own slices (26-connected, neighbours outside the slab
  // ignored) and ships the union-find parents with the labels; after the gather every rank only links the slab
  // boundaries and flattens
  const bool want_post = !(flags & LM_FLAG_NO_POSTPROCESS);
  const bool slab_ccl = want_post && e->shard_slab_ccl;
  uint32_t* parents_full = reinterpret_cast<uint32_t*>(v.block[v.rank] + shard_parents_offset(v.slice_cap, rr));
  const int vworld = (v.world == 1 && e->shard_test_slabs > 1) ? e->shard_test_slabs : v.world;   // test hook: virtual slabs on one GPU
  if (slab_ccl) {
    if (vworld == v.world) {
      if (ns > 0) RC(ccl_slab_device(labels_full, parents_full, S, R, R, lo, hi, e->post.ccl_rule, e->num_sms, e->st, &e->launches));
    } else {
      for (int r2 = 0; r2 < vworld; ++r2) {
        int l2, h2;
        shard_range(S, r2, vworld, &l2, &h2);
        RC(ccl_slab_device(labels_full, parents_full, S, R, R, l2, h2, e->post.ccl_rule, e->num_sms, e->st, &e->launches));
      }
    }
  }
  // the collective: wait until the peers have consumed the previous volume, push the slab, wait for theirs
  RC(launch_shard_wait_done(v, epoch, e->st));
  RC(launch_shard_push(v, (size_t)lo, (size_t)hi, rr, slab_ccl, epoch, e->num_sms, e->st));
  RC(launch_shard_wait_ready(v, epoch, e->st));
  e->launches += v.world > 1 ? 3 : 0;
  const uint8_t* masks = labels_full;
  if (want_post) {
    RC(e->d_post.reserve((size_t)S * rr));
    uint32_t* parent_in = nullptr;
    if (slab_ccl) {
      int firsts[kShardMaxWorld], nbounds = 0;
      for (int r2 = 1; r2 < vworld; ++r2) {
        int l2, h2;
        shard_range(S, r2, vworld, &l2, &h2);
        if (h2 > l2) firsts[nbounds++] = l2;
      }
      RC(ccl_join_slabs_device(labels_full, parents_full, S, R, R, firsts, nbounds, e->num_sms, e->st, &e->launches));
      parent_in = parents_full;
    }
    RC(postprocess_device(e->post, labels_full, S, R, R, nullptr, 0, nullptr, 0, 3, e->slots[slot].K - 1, e->d_post.p, e->num_sms, e->st,
                          &e->launches, parent_in));
    masks = e->d_post.p;
  }
  CU(cudaEventRecord(e->ev[4], e->st));
  RC(reshape_device(masks, boxes_full, S, H, W, R, R, d_out, e->num_sms, e->st));
  RC(launch_shard_signal_done(v, epoch, e->st));
  e->launches += v.world > 1 ? 2 : 1;
  CU(cudaEventRecord(e->ev[5], e->st));
  CU(cudaMemcpyAsync(e->h_shard_err, shard_error_word(v), sizeof(uint32_t), cudaMemcpyDeviceToHost, e->st));
  return 0;
}

int shard_check(lm_engine* e) {
  if (e->h_shard_err && *e->h_shard_err) {
    *e->h_shard_err = 0;
    cudaMemsetAsync(shard_error_word(e->shard), 0, sizeof(uint32_t), e->st);
    return fail(-50, "sharded gather: a peer rank did not arrive within the wait limit (rank %d of %d)", e->shard.rank, e->shard.world);
  }
  return 0;
}

void collect_timings(lm_engine* e) {
  if (e->time_convs) drain_conv_events(e);
  for (int i = 0; i < 6; ++i) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, e->ev[i], e->ev[i + 1]) != cudaSuccess) ms = -1.f;
    e->last_ms[i] = ms;
  }
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, e->ev[0], e->ev[6]) != cudaSuccess) ms = -1.f;
  e->last_ms[6] = ms;
}

// perm / flip of the oriented entry points -> pm / fl; both NULL: the identity (an LPS array).
int parse_orientation(const char* fn, const int* perm, const int* flip, int pm[3], int fl[3]) {
  for (int k = 0; k < 3; ++k) { pm[k] = k; fl[k] = 0; }
  if ((perm == nullptr) != (flip == nullptr)) return fail(-1, "%s: perm and flip must both be given or both be NULL", fn);
  if (!perm) return 0;
  int seen = 0;
  for (int k = 0; k < 3; ++k) {
    if (perm[k] < 0 || perm[k] > 2) return fail(-1, "%s: perm is not a permutation", fn);
    seen |= 1 << perm[k];
    pm[k] = perm[k];
    fl[k] = flip[k] != 0;
  }
  if (seen != 7) return fail(-1, "%s: perm is not a permutation", fn);
  return 0;
}

// A caller's pointer must be device (or managed) memory of the engine's device: a host pointer would fault in a kernel.
int check_device_ptr(const lm_engine* e, const char* fn, const char* what, const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return fail(-1, "%s: %s is not a CUDA pointer", fn, what);
  }
  if ((a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != e->device)
    return fail(-1, "%s: %s is not device memory of the engine's device %d", fn, what, e->device);
  return 0;
}

// The volume type inference_dev works in for an LM_DTYPE_* code: 0 int16, 1 float32, 2 float64.
int vtype_of(int dtype) {
  if (dtype == LM_DTYPE_F64) return 2;
  return (dtype == LM_DTYPE_F32 || dtype == LM_DTYPE_F16 || dtype == LM_DTYPE_BF16) ? 1 : 0;
}
size_t dtype_bytes(int dtype) {
  switch (dtype) {
    case LM_DTYPE_U8: case LM_DTYPE_I8: return 1;
    case LM_DTYPE_I16: case LM_DTYPE_F16: case LM_DTYPE_BF16: return 2;
    case LM_DTYPE_F32: case LM_DTYPE_I32: return 4;
    default: return 8;
  }
}

// One volume of LMInferer._inference / LMInferer.apply on device memory: the volume in its native orientation in, the
// mask (and the probabilities) in that orientation out.  Every whole-volume entry point runs one through run_volume,
// the _dev ones on the caller's pointers, the host ones on the engine buffers run_volume copies through.
struct VolumeJob {
  int slot, slot_fill;   // slot_fill >= 0: the fusion of mask.py:223-232
  const void* d_vol;     // (n0,n1,n2), element type `dtype` (LM_DTYPE_*); never written
  int dtype, flags;
  int dn[3], perm[3], flip[3];   // native dims; lps = transpose(native, perm) flipped along every axis k with flip[k]
  uint8_t* d_out;        // (n0,n1,n2)
  float* d_probs;        // nullptr, or (K,n0,n1,n2); not with slot_fill >= 0
};

// Enqueues the whole volume on the engine stream; the caller records ev[0] before and ev[6] after it.
int volume_enqueue(lm_engine* e, const VolumeJob& j) {
  const int* pm = j.perm;
  const int* fl = j.flip;
  const bool lps = pm[0] == 0 && pm[1] == 1 && pm[2] == 2 && !fl[0] && !fl[1] && !fl[2];
  const int dl[3] = {j.dn[pm[0]], j.dn[pm[1]], j.dn[pm[2]]};   // the LPS array: (slices, rows, columns) of the path
  const size_t n = (size_t)j.dn[0] * j.dn[1] * j.dn[2];
  const int vtype = vtype_of(j.dtype);
  const bool path_dtype = j.dtype == LM_DTYPE_I16 || j.dtype == LM_DTYPE_F32 || j.dtype == LM_DTYPE_F64;
  const void* d_lps_in = j.d_vol;   // an LPS volume of a path dtype is read in place
  if (!lps || !path_dtype) {
    // sitk.DICOMOrient(image, "LPS") (mask.py:163) and / or the dtype conversion of mask.py _to_engine_volume, one pass
    void* stage = nullptr;
    if (vtype == 0) { RC(e->d_vol.reserve(n)); stage = e->d_vol.p; }
    else { RC(e->d_fvol.reserve(n * (vtype == 2 ? 8 : 4))); stage = e->d_fvol.p; }
    RC(launch_orient_convert(j.d_vol, j.dtype, stage, dl, pm, fl, e->num_sms, e->st));
    e->launches++;
    d_lps_in = stage;
  }
  if (!lps) RC(e->d_lps_out.reserve(n));
  if (j.slot_fill < 0) {
    ProbOut po{nullptr, j.d_probs, {pm[0], pm[1], pm[2]}, {fl[0], fl[1], fl[2]}};
    if (j.d_probs) {
      RC(e->d_scores.reserve((size_t)dl[0] * e->slots[j.slot].K * R * R));
      po.scores = e->d_scores.p;
    }
    RC(inference_dev(e, j.slot, d_lps_in, vtype, dl[0], dl[1], dl[2], j.flags, lps ? j.d_out : e->d_lps_out.p,
                     j.d_probs ? &po : nullptr));
    if (!lps) {   // the mask back to the native orientation, mask.py:204-208
      RC(launch_orient_u8(e->d_lps_out.p, j.d_out, dl, pm, fl, 0, e->num_sms, e->st));
      e->launches++;
    }
    return 0;
  }
  // both inner inferences honour volume_postprocessing (mask.py:191-194); the fusion post-processing does not.  Each
  // _inference call re-orients its own result back, and the fusion and its post-processing work on the NATIVE-orientation
  // results (mask.py:225-232).
  const int inner = j.flags & LM_FLAG_NO_POSTPROCESS;
  RC(e->d_native_l.reserve(n));
  RC(e->d_native_r.reserve(n));
  const int slots[2] = {j.slot, j.slot_fill};
  uint8_t* const res[2] = {e->d_native_l.p, e->d_native_r.p};   // res_l, res_r (mask.py:225,227)
  for (int m = 0; m < 2; ++m) {
    RC(inference_dev(e, slots[m], d_lps_in, vtype, dl[0], dl[1], dl[2], inner, lps ? res[m] : e->d_lps_out.p, nullptr));
    if (!lps) {
      RC(launch_orient_u8(e->d_lps_out.p, res[m], dl, pm, fl, 0, e->num_sms, e->st));
      e->launches++;
    }
  }
  RC(fuse_device(res[0], res[1], n, e->d_scratch.p, e->d_spare, e->num_sms, e->st));   // spare stays on the device
  e->launches += 3;
  // labels after the fusion are <= K_base (the spare value is max + 1 <= K_base): mask.py:232
  RC(postprocess_device(e->post, res[0], j.dn[0], j.dn[1], j.dn[2], nullptr, 0, e->d_spare, 1, 3, e->slots[j.slot].K, j.d_out,
                        e->num_sms, e->st, &e->launches));
  return 0;
}

// The argument checks of the whole-volume entry points, with fn's name in the messages: -1 for a NULL pointer (ptrs_ok
// false) or an empty volume, -30 for a weight slot that is not loaded.  slot_fill < 0 means "no fill model", unless
// fill_required (lm_apply_fused*): there it is an unloaded slot as well.
int check_volume_call(const lm_engine* e, const char* fn, bool ptrs_ok, int n0, int n1, int n2, int slot, int slot_fill,
                      bool fill_required = false) {
  if (!e || !ptrs_ok) return fail(-1, "%s: NULL argument", fn);
  if (n0 < 1 || n1 < 1 || n2 < 1) return fail(-1, "%s: empty volume (%d,%d,%d)", fn, n0, n1, n2);
  if (slot < 0 || slot >= LM_MAX_SLOTS || !e->slots[slot].loaded) return fail(-30, "%s: weight slot %d not loaded", fn, slot);
  if ((slot_fill >= 0 || fill_required) && (slot_fill < 0 || slot_fill >= LM_MAX_SLOTS || !e->slots[slot_fill].loaded))
    return fail(-30, "%s: weight slot %d not loaded", fn, slot_fill);
  return 0;
}

// Runs one VolumeJob as a whole call: volume_enqueue between ev[0] and ev[6] under run_checked, then the timings.
//   h_vol    NULL (j.d_vol is device memory), or a host volume of j.dtype: uploaded to d_upload, which becomes j.d_vol.
//   h_out    NULL (j.d_out is device memory), or the host mask: copied back from d_out, which becomes j.d_out.
//   h_probs  NULL, or the host (K, n0, n1, n2) probabilities (needs h_out): copied back from d_out behind the mask.
//   caller   NULL, or the caller's stream: the engine stream waits for the work queued on it (lm_apply_dev).
int run_volume(lm_engine* e, VolumeJob j, const void* h_vol, uint8_t* h_out, float* h_probs, const cudaStream_t* caller = nullptr) {
  CU(cudaSetDevice(e->device));
  const size_t n = (size_t)j.dn[0] * j.dn[1] * j.dn[2], in_bytes = n * dtype_bytes(j.dtype);
  const size_t probs_at = (n + 255) & ~(size_t)255;
  const size_t probs_bytes = h_probs ? (size_t)e->slots[j.slot].K * n * sizeof(float) : 0;
  if (h_vol) {
    RC(e->d_upload.reserve(in_bytes));
    j.d_vol = e->d_upload.p;
  }
  if (h_out) {
    RC(e->d_out.reserve(h_probs ? probs_at + probs_bytes : n));
    j.d_out = e->d_out.p;
    if (h_probs) j.d_probs = reinterpret_cast<float*>(e->d_out.p + probs_at);
  }
  if (caller) CU(cudaEventRecord(e->ev_in, *caller));
  RC(run_checked(e, [&]() -> int {
    e->launches = 0;
    e->ev_used = 0;
    CU(cudaEventRecord(e->ev[0], e->st));
    if (caller) CU(cudaStreamWaitEvent(e->st, e->ev_in, 0));
    if (h_vol) CU(cudaMemcpyAsync(e->d_upload.p, h_vol, in_bytes, cudaMemcpyHostToDevice, e->st));
    RC(volume_enqueue(e, j));
    if (h_out) CU(cudaMemcpyAsync(h_out, j.d_out, n, cudaMemcpyDeviceToHost, e->st));
    if (h_probs) CU(cudaMemcpyAsync(h_probs, j.d_probs, probs_bytes, cudaMemcpyDeviceToHost, e->st));
    CU(cudaEventRecord(e->ev[6], e->st));
    return 0;
  }));
  collect_timings(e);
  return 0;
}

// A device pointer argument of an analysis call, with its name for the messages.
struct DevArg {
  const char* name;
  const void* p;
};

// The start of an analysis call (lm_label_stats_dev, lm_laa_clusters_dev, lm_plane_label_counts_dev,
// lm_surface_distance_dev, lm_region_map_dev, the texture and the shape calls), once its other arguments are checked: each device pointer must be memory
// of the engine's device (a NULL one is an optional input the call does not use), the engine's stream waits for the work
// queued on the caller's, and the launch count restarts.
int analysis_inputs(lm_engine* e, const char* fn, void* stream, std::initializer_list<DevArg> ptrs) {
  CU(cudaSetDevice(e->device));
  for (const DevArg& a : ptrs)
    if (a.p) RC(check_device_ptr(e, fn, a.name, a.p));
  CU(cudaEventRecord(e->ev_in, static_cast<cudaStream_t>(stream)));
  CU(cudaStreamWaitEvent(e->st, e->ev_in, 0));
  e->launches = 0;
  return 0;
}

}  // namespace

extern "C" {

const char* lm_last_error(void) { return g_err.c_str(); }
int lm_device(const lm_engine* e) { return e ? e->device : -1; }
int lm_batch_capacity(const lm_engine* e) { return e ? e->B : 0; }
size_t lm_weight_blob_floats(int n_classes) { return blob_floats(n_classes); }

static int create_resources(lm_engine* e);

int lm_create(int device, int batch_capacity, lm_engine** out) {
  if (!out) return fail(-1, "lm_create: out is NULL");
  *out = nullptr;
  if (batch_capacity < 1 || batch_capacity > 1024) return fail(-1, "lm_create: batch_capacity %d out of range", batch_capacity);
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0)
    return fail(ce ? (int)ce : -2, "lm_create: no CUDA device (%s); this engine has no CPU path", cudaGetErrorString(ce));
  if (device < 0 || device >= ndev) return fail(-1, "lm_create: device %d not in [0,%d)", device, ndev);
  CU(cudaSetDevice(device));
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(-3, "lm_create: device %s is sm_%d%d; this build is sm_90a only", prop.name, prop.major, prop.minor);
  lm_engine* e = new lm_engine();
  e->device = device;
  e->B = batch_capacity;
  e->num_sms = prop.multiProcessorCount;
  const int rc = create_resources(e);
  if (rc) {  // nothing of a half-built engine survives a failed create (the message of the failing call is kept)
    const std::string msg = g_err;
    lm_destroy(e);
    cudaGetLastError();
    g_err = msg;
    return rc;
  }
  *out = e;
  return 0;
}

static int create_resources(lm_engine* e) {
  const int batch_capacity = e->B;
  if (const char* c = getenv("LM_CHUNK_KB")) { int v = atoi(c); if (v >= 1) e->chunk_kb = e->chunk_kb_wide = v; }
  if (const char* c = getenv("LM_WEIGHT_MCAST")) e->weight_mcast = atoi(c) == 2 ? 2 : 0;
  if (const char* c = getenv("LM_CONV64_CM")) e->conv64_cm = atoi(c) != 0;
  if (const char* c = getenv("LM_GRAPHS")) e->use_graphs = atoi(c) != 0;
  if (const char* c = getenv("LM_BN64_MASK")) e->bn64_mask = (unsigned)strtoul(c, nullptr, 0);
  if (const char* c = getenv("LM_STEM_V2")) { const int v = atoi(c); e->stem_v2 = v < 0 ? 0 : (v > 3 ? 3 : v); }
  if (const char* c = getenv("LM_UPSAMPLE_V2")) { const int v = atoi(c); e->upsample_v2 = v < 0 ? 0 : (v > 2 ? 2 : v); }
  if (const char* c = getenv("LM_CCL_RULE")) e->post.ccl_rule = atoi(c) != 0;
  if (const char* c = getenv("LM_MERGE_CTAS")) e->post.merge_ctas = atoi(c) > 0 ? atoi(c) : 0;
  if (const char* c = getenv("LM_CHUNK_KB_WIDE")) { int v = atoi(c); if (v >= 1) e->chunk_kb_wide = v; }
  RC(conv_tc_prepare());
  CU(cudaStreamCreateWithFlags(&e->st, cudaStreamNonBlocking));
  for (int i = 0; i < 8; ++i) CU(cudaEventCreate(&e->ev[i]));
  for (int i = 0; i < 2; ++i) CU(cudaEventCreate(&e->ev_conv[i]));
  CU(cudaEventCreateWithFlags(&e->ev_in, cudaEventDisableTiming));
  for (int a = 0; a < NUM_ACT; ++a) {
    const int hw = R >> ACT[a].level;
    const size_t elems = (size_t)batch_capacity * hw * hw * ACT[a].C;
    CU(cudaMalloc(&e->act[a], ACT[a].split ? elems * 2 * sizeof(op_t) : elems * sizeof(float)));
  }
  CU(cudaMalloc(&e->d_spare, 16 * sizeof(int32_t)));
  CU(cudaMalloc(&e->d_range, LM_MAX_SLOTS * RANGE_STRIDE * sizeof(int)));
  CU(cudaMemset(e->d_range, 0, LM_MAX_SLOTS * RANGE_STRIDE * sizeof(int)));
  CU(cudaMallocHost(&e->h_range, LM_MAX_SLOTS * RANGE_STRIDE * sizeof(int)));
  memset(e->h_range, 0, LM_MAX_SLOTS * RANGE_STRIDE * sizeof(int));
  RC(e->d_scratch.reserve(64));
  return 0;
}

void lm_destroy(lm_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaStreamSynchronize(e->st);
  drop_graphs(e);
  for (int a = 0; a < NUM_ACT; ++a) cudaFree(e->act[a]);
  shard_release(e);
  cudaFree(e->d_range);
  cudaFree(e->d_spare);
  cudaFreeHost(e->h_range);
  for (auto& s : e->slots) {
    cudaFree(s.stem_w); cudaFree(s.stem_bias); cudaFree(s.stem_scale); cudaFree(s.stem_shift); cudaFree(s.head_w); cudaFree(s.head_b);
    for (auto& l : s.lw) { cudaFree(l.w); cudaFree(l.bias); cudaFree(l.scale); cudaFree(l.shift); }
  }
  e->d_norm.release(); e->d_fvol.release(); e->d_upload.release();
  e->d_lps_out.release(); e->d_native_l.release(); e->d_native_r.release();
  e->d_vol.release(); e->d_resized.release(); e->d_boxes.release(); e->d_labels.release(); e->d_post.release();
  e->d_out.release(); e->d_out2.release(); e->d_mask.release(); e->d_scores.release(); e->d_scratch.release();
  e->post.release();
  e->stats.release();
  e->clusters.release();
  e->regions.release();
  e->texture.release();
  e->shape.release();
  e->first_order.release();
  e->wavelet.release();
  e->filters.release();
  e->mesh.release();
  e->fo_maps.release();
  e->glcm_maps.release();
  e->texture_maps.release();
  e->resample.release();
  e->laplacian.release();
  for (auto& ev : e->ev) cudaEventDestroy(ev);
  for (auto& ev : e->ev_conv) cudaEventDestroy(ev);
  for (auto& ev : e->ev_pool) cudaEventDestroy(ev);
  if (e->ev_in) cudaEventDestroy(e->ev_in);
  cudaStreamDestroy(e->st);
  delete e;
}

int lm_load_weights(lm_engine* e, int slot, const float* blob, size_t n_floats, int K) {
  if (!e || !blob) return fail(-1, "lm_load_weights: NULL argument");
  if (slot < 0 || slot >= LM_MAX_SLOTS) return fail(-1, "lm_load_weights: slot %d out of range", slot);
  if (K < 1 || K > 8) return fail(-1, "lm_load_weights: n_classes %d not in [1,8]", K);
  if (n_floats != blob_floats(K)) return fail(-1, "lm_load_weights: blob has %zu floats, expected %zu for %d classes", n_floats, blob_floats(K), K);
  CU(cudaSetDevice(e->device));
  Slot& s = e->slots[slot];
  s.loaded = false;
  s.K = K;
  e->graph_epoch++;
  const float* q = blob;
  std::vector<float> scale, shift;
  struct Tmp {  // staging buffer for one layer's OIHW weights (largest: 1024 x 1024 x 9), freed on every exit path
    float* p = nullptr;
    ~Tmp() { if (p) cudaFree(p); }
  } tmp;
  CU(cudaMalloc(&tmp.p, (size_t)1024 * 1024 * 9 * sizeof(float)));
  float* const d_tmp = tmp.p;
  // stem
  RC(upload(&s.stem_w, q, 64 * 9, e->st)); q += 64 * 9;
  RC(upload(&s.stem_bias, q, 64, e->st)); q += 64;
  fold_bn(q, q + 64, q + 128, q + 192, 64, scale, shift); q += 256;
  RC(upload(&s.stem_scale, scale.data(), 64, e->st));
  RC(upload(&s.stem_shift, shift.data(), 64, e->st));
  auto load_conv = [&](int i, bool has_bn) -> int {
    const LayerSpec& L = LAYERS[i];
    const int Cin = L.C0 + L.C1;
    const size_t nw = (size_t)L.Cout * Cin * L.taps;
    // power-of-two weight scale (undone, exactly, by ConvParams::in_unscale); non-finite weights are refused
    float wmax = 0.f;
    for (size_t k = 0; k < nw; ++k) {
      const float a = fabsf(q[k]);
      if (!(a <= 3.0e38f)) return fail(LM_ERR_RANGE, "lm_load_weights: layer %d holds a non-finite weight", i);
      wmax = a > wmax ? a : wmax;
    }
    // normalise the layer to the top of the operand format's range, max |w| * ws in (2^14, 2^15]: the hi / lo planes then
    // keep their 11 + 11 bits for every weight down to 2^-28 of the largest one, whatever the layer's magnitude
    float ws = 1.f;
    if (wmax > 0.f) {
      while (wmax * ws > 32768.f) ws *= 0.5f;
      while (wmax * ws <= 16384.f && ws < 1.0e30f) ws *= 2.f;
    }
    s.lw[i].w_scale = ws;
    CU(cudaMemcpyAsync(d_tmp, q, nw * sizeof(float), cudaMemcpyHostToDevice, e->st)); q += nw;
    if (!s.lw[i].w) CU(cudaMalloc(&s.lw[i].w, 2 * nw * sizeof(op_t)));
    RC(launch_prep_conv_weights(d_tmp, s.lw[i].w, L.Cout, Cin, L.taps, e->d_range + slot * RANGE_STRIDE + NUM_ACT, ws, e->st));
    CU(cudaStreamSynchronize(e->st));
    RC(upload(&s.lw[i].bias, q, L.Cout, e->st)); q += L.Cout;
    if (has_bn) {
      fold_bn(q, q + L.Cout, q + 2 * L.Cout, q + 3 * L.Cout, L.Cout, scale, shift); q += 4 * L.Cout;
    } else {
      scale.assign(L.Cout, 1.f); shift.assign(L.Cout, 0.f);
    }
    RC(upload(&s.lw[i].scale, scale.data(), L.Cout, e->st));
    RC(upload(&s.lw[i].shift, shift.data(), L.Cout, e->st));
    return 0;
  };
  for (int i = 0; i < NUM_LAYERS; ++i) if (LAYERS[i].taps == 9) RC(load_conv(i, true));
  for (int i = 0; i < NUM_LAYERS; ++i) if (LAYERS[i].taps == 1) RC(load_conv(i, false));
  cudaFree(s.head_w); cudaFree(s.head_b);  // sized by the class count of the previous load
  s.head_w = s.head_b = nullptr;
  RC(upload(&s.head_w, q, (size_t)K * 64, e->st)); q += (size_t)K * 64;
  RC(upload(&s.head_b, q, K, e->st)); q += K;
  if ((size_t)(q - blob) != n_floats) return fail(-1, "lm_load_weights: internal blob walk mismatch");
  int* const h_wflag = e->h_range + slot * RANGE_STRIDE + NUM_ACT;
  CU(cudaMemcpyAsync(h_wflag, e->d_range + slot * RANGE_STRIDE + NUM_ACT, sizeof(int), cudaMemcpyDeviceToHost, e->st));
  CU(cudaStreamSynchronize(e->st));
  if (*h_wflag) {
    *h_wflag = 0;
    CU(cudaMemsetAsync(e->d_range + slot * RANGE_STRIDE + NUM_ACT, 0, sizeof(int), e->st));
    return fail(LM_ERR_RANGE, "lm_load_weights: a scaled convolution weight still exceeds the fp16 operand range (internal error)");
  }
  for (float& sc : s.act_scale) sc = 1.f;   // new weights: activation ranges are unknown again
  for (int i = 0; i < NUM_LAYERS; ++i) {
    const LayerSpec& L = LAYERS[i];
    ConvParams p{};
    p.N = e->B; p.H = R >> L.level; p.W = R >> L.level; p.C0 = L.C0; p.C1 = L.C1; p.Cout = L.Cout; p.taps = L.taps;
    p.mode = L.mode; p.chunk_kb = e->chunk_kb;
    p.bias = s.lw[i].bias; p.scale = s.lw[i].scale; p.shift = s.lw[i].shift;
    p.out = L.dst >= 0 ? e->act[L.dst] : nullptr;
    p.out_pool = L.dst_pool >= 0 ? e->act[L.dst_pool] : nullptr;
    p.head_w = s.head_w; p.head_b = s.head_b; p.K = K;
    p.tile_n = ((e->bn64_mask >> i) & 1u) ? 64 : 0;
    s.params[i] = p;
    int r = make_conv_maps(&s.maps[i], e->act[L.src0], L.src1 >= 0 ? e->act[L.src1] : nullptr, s.lw[i].w, p, e->B);
    if (r) return fail(r, "make_conv_maps failed for layer %d: %d", i, r);
  }
  s.loaded = true;
  return 0;
}

int lm_apply_volume_dev(lm_engine* e, int slot, const int16_t* d_vol, int S, int H, int W, int flags, uint8_t* d_out) {
  RC(check_volume_call(e, "lm_apply_volume_dev", d_vol && d_out, S, H, W, slot, -1));
  return run_volume(e, {slot, -1, d_vol, LM_DTYPE_I16, flags, {S, H, W}, {0, 1, 2}, {0, 0, 0}, d_out, nullptr}, nullptr, nullptr,
                    nullptr);
}

int lm_apply_volume(lm_engine* e, int slot, const int16_t* vol, int S, int H, int W, int flags, uint8_t* out) {
  RC(check_volume_call(e, "lm_apply_volume", vol && out, S, H, W, slot, -1));
  return run_volume(e, {slot, -1, nullptr, LM_DTYPE_I16, flags, {S, H, W}, {0, 1, 2}, {0, 0, 0}, nullptr, nullptr}, vol, out,
                    nullptr);
}

int lm_apply_fused(lm_engine* e, int slot_base, int slot_fill, const int16_t* vol, int S, int H, int W, int flags, uint8_t* out) {
  RC(check_volume_call(e, "lm_apply_fused", vol && out, S, H, W, slot_base, slot_fill, true));
  return run_volume(e, {slot_base, slot_fill, nullptr, LM_DTYPE_I16, flags, {S, H, W}, {0, 1, 2}, {0, 0, 0}, nullptr, nullptr},
                    vol, out, nullptr);
}

int lm_apply_fused_dev(lm_engine* e, int slot_base, int slot_fill, const int16_t* d_vol, int S, int H, int W, int flags, uint8_t* d_out) {
  RC(check_volume_call(e, "lm_apply_fused_dev", d_vol && d_out, S, H, W, slot_base, slot_fill, true));
  return run_volume(e, {slot_base, slot_fill, d_vol, LM_DTYPE_I16, flags, {S, H, W}, {0, 1, 2}, {0, 0, 0}, d_out, nullptr},
                    nullptr, nullptr, nullptr);
}

int lm_apply_volume_float(lm_engine* e, int slot, int slot_fill, const void* vol, int is_f64, int S, int H, int W, int flags,
                          uint8_t* out) {
  RC(check_volume_call(e, "lm_apply_volume_float", vol && out, S, H, W, slot, slot_fill));
  const int dtype = is_f64 ? LM_DTYPE_F64 : LM_DTYPE_F32;
  return run_volume(e, {slot, slot_fill, nullptr, dtype, flags, {S, H, W}, {0, 1, 2}, {0, 0, 0}, nullptr, nullptr}, vol, out,
                    nullptr);
}

int lm_preprocess_float(lm_engine* e, const void* vol, int is_f64, int S, int H, int W, float* normalised, int32_t* boxes) {
  if (!e || !vol || !normalised || !boxes) return fail(-1, "lm_preprocess_float: NULL argument");
  if (S < 1 || H < 1 || W < 1) return fail(-1, "lm_preprocess_float: empty volume");
  CU(cudaSetDevice(e->device));
  const size_t n = (size_t)S * H * W, esz = is_f64 ? 8 : 4, nr = (size_t)S * R * R;
  RC(e->d_fvol.reserve(n * esz));
  RC(e->d_boxes.reserve((size_t)S * 4));
  RC(e->d_norm.reserve(nr));
  CU(cudaMemcpyAsync(e->d_fvol.p, vol, n * esz, cudaMemcpyHostToDevice, e->st));
  RC(launch_bodymask_float(e->d_fvol.p, is_f64, S, H, W, e->d_boxes.p, nullptr, e->num_sms, e->st));
  RC(launch_resize_float(e->d_fvol.p, is_f64, S, H, W, e->d_boxes.p, e->d_norm.p, R, R, e->num_sms, e->st));
  CU(cudaMemcpyAsync(normalised, e->d_norm.p, nr * sizeof(float), cudaMemcpyDeviceToHost, e->st));
  CU(cudaMemcpyAsync(boxes, e->d_boxes.p, (size_t)S * 4 * sizeof(int32_t), cudaMemcpyDeviceToHost, e->st));
  CU(cudaStreamSynchronize(e->st));
  return 0;
}

int lm_apply_volume_oriented(lm_engine* e, int slot, int slot_fill, const int16_t* vol, int n0, int n1, int n2, const int* perm,
                             const int* flip, int flags, uint8_t* out) {
  RC(check_volume_call(e, "lm_apply_volume_oriented", vol && out && perm && flip, n0, n1, n2, slot, slot_fill));
  VolumeJob j{slot, slot_fill, nullptr, LM_DTYPE_I16, flags, {n0, n1, n2}, {}, {}, nullptr, nullptr};
  RC(parse_orientation("lm_apply_volume_oriented", perm, flip, j.perm, j.flip));
  return run_volume(e, j, vol, out, nullptr);
}

int lm_apply_volume_probs(lm_engine* e, int slot, const void* vol, int dtype, int n0, int n1, int n2, const int* perm,
                          const int* flip, int flags, uint8_t* out, float* probs) {
  RC(check_volume_call(e, "lm_apply_volume_probs", vol && out && probs, n0, n1, n2, slot, -1));
  if (dtype != LM_DTYPE_I16 && dtype != LM_DTYPE_F32 && dtype != LM_DTYPE_F64)
    return fail(-1, "lm_apply_volume_probs: dtype %d is not LM_DTYPE_I16, LM_DTYPE_F32 or LM_DTYPE_F64", dtype);
  VolumeJob j{slot, -1, nullptr, dtype, flags, {n0, n1, n2}, {}, {}, nullptr, nullptr};
  RC(parse_orientation("lm_apply_volume_probs", perm, flip, j.perm, j.flip));
  return run_volume(e, j, vol, out, probs);
}

int lm_apply_dev(lm_engine* e, int slot, int slot_fill, const void* d_vol, int dtype, int n0, int n1, int n2, const int* perm,
                 const int* flip, int flags, uint8_t* d_out, float* d_probs, void* stream) {
  RC(check_volume_call(e, "lm_apply_dev", d_vol && d_out, n0, n1, n2, slot, slot_fill));
  if (dtype < LM_DTYPE_I16 || dtype > LM_DTYPE_BF16) return fail(-1, "lm_apply_dev: unknown dtype code %d", dtype);
  VolumeJob j{slot, slot_fill, d_vol, dtype, flags, {n0, n1, n2}, {}, {}, d_out, d_probs};
  RC(parse_orientation("lm_apply_dev", perm, flip, j.perm, j.flip));
  if (slot_fill >= 0 && d_probs)
    return fail(-1, "lm_apply_dev: no probabilities for the fusion with a fill model (slot_fill %d): the reference's fusion "
                    "defines none", slot_fill);
  CU(cudaSetDevice(e->device));
  RC(check_device_ptr(e, "lm_apply_dev", "d_vol", d_vol));
  RC(check_device_ptr(e, "lm_apply_dev", "d_out", d_out));
  if (d_probs) RC(check_device_ptr(e, "lm_apply_dev", "d_probs", d_probs));
  const cudaStream_t caller = static_cast<cudaStream_t>(stream);
  return run_volume(e, j, nullptr, nullptr, nullptr, &caller);
}

int lm_label_stats_dev(lm_engine* e, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2,
                       const double* percentiles, int n_q, const int* thresholds, int n_t, int64_t* voxels,
                       int64_t* nan_voxels, double* moments, double* percentile, int64_t* below_count, void* stream) {
  static const char* fn = "lm_label_stats_dev";
  const double* q = percentiles;
  const int* t = thresholds;
  if (!e || !d_vol || !d_mask || !voxels || !nan_voxels || !moments || (n_q > 0 && (!q || !percentile)) ||
      (n_t > 0 && (!t || !below_count)))
    return fail(-1, "%s: NULL argument", fn);
  if (n0 < 1 || n1 < 1 || n2 < 1) return fail(-1, "%s: empty volume (%d,%d,%d)", fn, n0, n1, n2);
  if (dtype < LM_DTYPE_I16 || dtype > LM_DTYPE_BF16) return fail(-1, "%s: unknown dtype code %d", fn, dtype);
  if (n_q < 0 || n_q > LM_STATS_MAX_PERCENTILES) return fail(-1, "%s: n_q %d not in [0,%d]", fn, n_q, LM_STATS_MAX_PERCENTILES);
  if (n_t < 0 || n_t > LM_STATS_MAX_THRESHOLDS) return fail(-1, "%s: n_t %d not in [0,%d]", fn, n_t, LM_STATS_MAX_THRESHOLDS);
  for (int k = 0; k < n_q; ++k)
    if (!(q[k] >= 0.0 && q[k] <= 100.0)) return fail(-1, "%s: percentile %g not in [0,100]", fn, q[k]);
  for (int k = 0; k < n_t; ++k)
    if (t[k] < -1024 || t[k] > 3072) return fail(-1, "%s: threshold %d not in [-1024,3072]", fn, t[k]);
  RC(analysis_inputs(e, fn, stream, {{"d_vol", d_vol}, {"d_mask", d_mask}}));
  const LabelStatsOut out{voxels, nan_voxels, moments, percentile, below_count};
  RC(label_stats(e->stats, d_vol, dtype, d_mask, (size_t)n0 * n1 * n2, q, n_q, t, n_t, out, e->num_sms, e->st, &e->launches));
  return 0;
}

size_t lm_laa_max_pairs(size_t n_voxels) { return laa_max_pairs(n_voxels); }

int lm_laa_clusters_dev(lm_engine* e, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2, int threshold,
                        int connectivity, int64_t* laa_voxels, int64_t* n_clusters, int64_t* n_pairs, int64_t* sizes,
                        int64_t* counts, size_t max_pairs, void* stream) {
  static const char* fn = "lm_laa_clusters_dev";
  if (!e || !d_vol || !d_mask || !laa_voxels || !n_clusters || !n_pairs || !sizes || !counts)
    return fail(-1, "%s: NULL argument", fn);
  if (n0 < 1 || n1 < 1 || n2 < 1) return fail(-1, "%s: empty volume (%d,%d,%d)", fn, n0, n1, n2);
  const size_t n = (size_t)n0 * n1 * n2;
  if (n >= ((size_t)1 << 32)) return fail(-1, "%s: %zu voxels, the labelling takes fewer than 2^32", fn, n);
  if (dtype < LM_DTYPE_I16 || dtype > LM_DTYPE_BF16) return fail(-1, "%s: unknown dtype code %d", fn, dtype);
  if (threshold < -1024 || threshold > 3072) return fail(-1, "%s: threshold %d not in [-1024,3072]", fn, threshold);
  if (connectivity != 4 && connectivity != 6 && connectivity != 26)
    return fail(-1, "%s: connectivity %d is not 4, 6 or 26", fn, connectivity);
  if (max_pairs < laa_max_pairs(n))
    return fail(-1, "%s: max_pairs %zu below lm_laa_max_pairs(%zu) = %zu", fn, max_pairs, n, laa_max_pairs(n));
  RC(analysis_inputs(e, fn, stream, {{"d_vol", d_vol}, {"d_mask", d_mask}}));
  const LaaClustersOut out{laa_voxels, n_clusters, n_pairs, sizes, counts, max_pairs};
  RC(laa_clusters(e->clusters, d_vol, dtype, d_mask, n0, n1, n2, threshold, connectivity, out, e->num_sms, e->st, &e->launches));
  return 0;
}

int lm_plane_label_counts_dev(lm_engine* e, const uint8_t* d_mask, int n0, int n1, int n2, int axis, int64_t* counts, void* stream) {
  static const char* fn = "lm_plane_label_counts_dev";
  if (!e || !d_mask || !counts) return fail(-1, "%s: NULL argument", fn);
  if (n0 < 1 || n1 < 1 || n2 < 1) return fail(-1, "%s: empty volume (%d,%d,%d)", fn, n0, n1, n2);
  if (axis < 0 || axis > 2) return fail(-1, "%s: axis %d is not 0, 1 or 2", fn, axis);
  RC(analysis_inputs(e, fn, stream, {{"d_mask", d_mask}}));
  RC(plane_label_counts(e->regions, d_mask, n0, n1, n2, axis, counts, e->num_sms, e->st, &e->launches));
  return 0;
}

int lm_surface_distance_dev(lm_engine* e, const uint8_t* d_mask, int n0, int n1, int n2, const double* spacing, float* d_out,
                            void* stream) {
  static const char* fn = "lm_surface_distance_dev";
  if (!e || !d_mask || !spacing || !d_out) return fail(-1, "%s: NULL argument", fn);
  if (n0 < 1 || n1 < 1 || n2 < 1) return fail(-1, "%s: empty volume (%d,%d,%d)", fn, n0, n1, n2);
  for (int k = 0; k < 3; ++k)
    if (!(spacing[k] > 0.0 && spacing[k] < INFINITY)) return fail(-1, "%s: spacing[%d] = %g is not finite and positive", fn, k, spacing[k]);
  if (n0 >= (1 << 30) || n1 >= (1 << 30) || n2 >= (1 << 30)) return fail(-1, "%s: (%d,%d,%d): an axis of 2^30 or more", fn, n0, n1, n2);
  RC(analysis_inputs(e, fn, stream, {{"d_mask", d_mask}, {"d_out", d_out}}));
  RC(surface_distance(e->regions, d_mask, n0, n1, n2, spacing, d_out, e->num_sms, e->st, &e->launches));
  CU(cudaStreamSynchronize(e->st));
  return 0;
}

int lm_region_map_dev(lm_engine* e, const uint8_t* d_mask, const float* d_dist, int n0, int n1, int n2, int axis,
                      const float* bounds, int n_bounds, const uint8_t* lut, size_t lut_size, uint8_t* d_map, void* stream) {
  static const char* fn = "lm_region_map_dev";
  if (!e || !d_mask || !lut || !d_map || (d_dist && n_bounds > 0 && !bounds)) return fail(-1, "%s: NULL argument", fn);
  if (n0 < 1 || n1 < 1 || n2 < 1) return fail(-1, "%s: empty volume (%d,%d,%d)", fn, n0, n1, n2);
  size_t buckets;
  if (d_dist) {
    if (n_bounds < 0 || n_bounds > 254) return fail(-1, "%s: n_bounds %d not in [0,254]", fn, n_bounds);
    for (int k = 0; k < n_bounds; ++k) {
      if (!(bounds[k] > 0.0f && bounds[k] < INFINITY)) return fail(-1, "%s: bound %g is not finite and positive", fn, bounds[k]);
      if (k > 0 && !(bounds[k] > bounds[k - 1])) return fail(-1, "%s: bounds are not strictly increasing", fn);
    }
    buckets = (size_t)n_bounds + 1;
  } else {
    if (axis < 0 || axis > 2) return fail(-1, "%s: axis %d is not 0, 1 or 2", fn, axis);
    if (n_bounds != 0) return fail(-1, "%s: shell bounds without d_dist", fn);
    buckets = (size_t)(axis == 0 ? n0 : (axis == 1 ? n1 : n2));
  }
  if (lut_size != buckets * 256) return fail(-1, "%s: lut_size %zu, expected %zu buckets x 256 = %zu", fn, lut_size, buckets, buckets * 256);
  for (size_t b = 0; b < buckets; ++b)
    if (lut[b * 256]) return fail(-1, "%s: lut[%zu][0] = %d, label 0 must map to 0", fn, b, (int)lut[b * 256]);
  RC(analysis_inputs(e, fn, stream, {{"d_mask", d_mask}, {"d_dist", d_dist}, {"d_map", d_map}}));
  RC(region_map(e->regions, d_mask, d_dist, n0, n1, n2, d_dist ? -1 : axis, bounds, d_dist ? n_bounds : 0, lut, lut_size, d_map,
                e->num_sms, e->st, &e->launches));
  return 0;
}

// The argument checks the texture calls share: the shape (fewer than 2^32 voxels).
static int check_texture_volume(const char* fn, int n0, int n1, int n2) {
  if (n0 < 1 || n1 < 1 || n2 < 1) return fail(-1, "%s: empty volume (%d,%d,%d)", fn, n0, n1, n2);
  const size_t n = (size_t)n0 * n1 * n2;
  if (n >= ((size_t)1 << 32)) return fail(-1, "%s: %zu voxels, the texture calls take fewer than 2^32", fn, n);
  return 0;
}

// A level outside 1..n_levels or a non-finite value found on the device.
static int texture_device_error(const char* fn, int rc, int n_levels) {
  if (rc == kLevelRange) return fail(rc, "%s: a level outside 1..%d (n_levels) in the ROI", fn, n_levels);
  if (rc == kLevelNonFinite) return fail(rc, "%s: a non-finite value (+-inf) in the ROI", fn);
  return rc;
}

int lm_texture_levels_dev(lm_engine* e, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2, int row,
                          int64_t low, int bin_width, int n_levels, uint8_t* d_levels, void* stream) {
  static const char* fn = "lm_texture_levels_dev";
  if (!e || !d_vol || !d_mask || !d_levels) return fail(-1, "%s: NULL argument", fn);
  RC(check_texture_volume(fn, n0, n1, n2));
  if (dtype < LM_DTYPE_I16 || dtype > LM_DTYPE_BF16) return fail(-1, "%s: unknown dtype code %d", fn, dtype);
  if (row < 1 || row > 256) return fail(-1, "%s: row %d not in [1,256]", fn, row);
  if (bin_width < 1) return fail(-1, "%s: bin_width %d is not positive", fn, bin_width);
  if (n_levels < 1 || n_levels > kTextureMaxLevels) return fail(-1, "%s: n_levels %d not in [1,%d]", fn, n_levels, kTextureMaxLevels);
  if (reinterpret_cast<uintptr_t>(d_levels) & 15) return fail(-1, "%s: d_levels is not 16-byte aligned", fn);
  RC(analysis_inputs(e, fn, stream, {{"d_vol", d_vol}, {"d_mask", d_mask}, {"d_levels", d_levels}}));
  const int rc = texture_levels(e->texture, d_vol, dtype, d_mask, (size_t)n0 * n1 * n2, row, low, bin_width, n_levels, d_levels,
                                e->num_sms, e->st, &e->launches);
  if (rc) return texture_device_error(fn, rc, n_levels);
  return 0;
}

int lm_glcm_dev(lm_engine* e, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int64_t* counts, void* stream) {
  static const char* fn = "lm_glcm_dev";
  if (!e || !d_levels || !counts) return fail(-1, "%s: NULL argument", fn);
  RC(check_texture_volume(fn, n0, n1, n2));
  if (n_levels < 1 || n_levels > kTextureMaxLevels) return fail(-1, "%s: n_levels %d not in [1,%d]", fn, n_levels, kTextureMaxLevels);
  RC(analysis_inputs(e, fn, stream, {{"d_levels", d_levels}}));
  const int rc = glcm(e->texture, d_levels, n0, n1, n2, n_levels, counts, e->num_sms, e->st, &e->launches);
  if (rc) return texture_device_error(fn, rc, n_levels);
  return 0;
}

int lm_glrlm_dev(lm_engine* e, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int64_t* counts, void* stream) {
  static const char* fn = "lm_glrlm_dev";
  if (!e || !d_levels || !counts) return fail(-1, "%s: NULL argument", fn);
  RC(check_texture_volume(fn, n0, n1, n2));
  if (n_levels < 1 || n_levels > kTextureMaxLevels) return fail(-1, "%s: n_levels %d not in [1,%d]", fn, n_levels, kTextureMaxLevels);
  RC(analysis_inputs(e, fn, stream, {{"d_levels", d_levels}}));
  const int rc = glrlm(e->texture, d_levels, n0, n1, n2, n_levels, counts, e->num_sms, e->st, &e->launches);
  if (rc) return texture_device_error(fn, rc, n_levels);
  return 0;
}

int lm_neighbour_counts_dev(lm_engine* e, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int alpha,
                            int64_t* dependence, int64_t* ngtdm_counts, int64_t* ngtdm_sums, void* stream) {
  static const char* fn = "lm_neighbour_counts_dev";
  if (!e || !d_levels || !dependence || !ngtdm_counts || !ngtdm_sums) return fail(-1, "%s: NULL argument", fn);
  RC(check_texture_volume(fn, n0, n1, n2));
  if (n_levels < 1 || n_levels > kTextureMaxLevels) return fail(-1, "%s: n_levels %d not in [1,%d]", fn, n_levels, kTextureMaxLevels);
  if (alpha < 0) return fail(-1, "%s: alpha %d is negative", fn, alpha);
  RC(analysis_inputs(e, fn, stream, {{"d_levels", d_levels}}));
  const int rc = neighbour_counts(e->texture, d_levels, n0, n1, n2, n_levels, alpha, dependence, ngtdm_counts, ngtdm_sums,
                                  e->num_sms, e->st, &e->launches);
  if (rc) return texture_device_error(fn, rc, n_levels);
  return 0;
}

int lm_zone_sizes_dev(lm_engine* e, const uint8_t* d_levels, int n0, int n1, int n2, int64_t* n_pairs, int64_t* sizes,
                      int64_t* counts, size_t max_pairs, void* stream) {
  static const char* fn = "lm_zone_sizes_dev";
  if (!e || !d_levels || !n_pairs || !sizes || !counts) return fail(-1, "%s: NULL argument", fn);
  RC(check_texture_volume(fn, n0, n1, n2));
  const size_t n = (size_t)n0 * n1 * n2;
  if (max_pairs < laa_max_pairs(n))
    return fail(-1, "%s: max_pairs %zu below lm_laa_max_pairs(%zu) = %zu", fn, max_pairs, n, laa_max_pairs(n));
  RC(analysis_inputs(e, fn, stream, {{"d_levels", d_levels}}));
  RC(zone_sizes(e->clusters, d_levels, n0, n1, n2, n_pairs, sizes, counts, max_pairs, e->num_sms, e->st, &e->launches));
  return 0;
}

// The offset list of lm_glcm_offsets_dev / lm_neighbour_offsets_dev: 1..171 distinct offsets, components in -3..3,
// Chebyshev norm >= 1, first non-zero component positive.
static int check_offsets(const char* fn, const int8_t* offsets, int n_offsets) {
  if (!offsets) return fail(-1, "%s: NULL offsets", fn);
  if (n_offsets < 1 || n_offsets > kMaxOffsets) return fail(-1, "%s: n_offsets %d not in [1,%d]", fn, n_offsets, kMaxOffsets);
  for (int k = 0; k < n_offsets; ++k) {
    const int dz = offsets[3 * k], dy = offsets[3 * k + 1], dx = offsets[3 * k + 2];
    if (dz < -3 || dz > 3 || dy < -3 || dy > 3 || dx < -3 || dx > 3)
      return fail(-1, "%s: offset %d (%d,%d,%d) has a component outside -3..3", fn, k, dz, dy, dx);
    const int first = dz ? dz : (dy ? dy : dx);
    if (first == 0) return fail(-1, "%s: offset %d is (0,0,0)", fn, k);
    if (first < 0) return fail(-1, "%s: offset %d (%d,%d,%d): the first non-zero component is negative", fn, k, dz, dy, dx);
    for (int j = 0; j < k; ++j)
      if (offsets[3 * j] == dz && offsets[3 * j + 1] == dy && offsets[3 * j + 2] == dx)
        return fail(-1, "%s: offset %d (%d,%d,%d) repeats offset %d", fn, k, dz, dy, dx, j);
  }
  return 0;
}

int lm_glcm_offsets_dev(lm_engine* e, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, const int8_t* offsets,
                        int n_offsets, int64_t* counts, void* stream) {
  static const char* fn = "lm_glcm_offsets_dev";
  if (!e || !d_levels || !counts) return fail(-1, "%s: NULL argument", fn);
  RC(check_offsets(fn, offsets, n_offsets));
  RC(check_texture_volume(fn, n0, n1, n2));
  if (n_levels < 1 || n_levels > kTextureMaxLevels) return fail(-1, "%s: n_levels %d not in [1,%d]", fn, n_levels, kTextureMaxLevels);
  RC(analysis_inputs(e, fn, stream, {{"d_levels", d_levels}}));
  const int rc = glcm_offsets(e->texture, d_levels, n0, n1, n2, n_levels, offsets, n_offsets, counts, e->num_sms, e->st,
                              &e->launches);
  if (rc) return texture_device_error(fn, rc, n_levels);
  return 0;
}

int lm_neighbour_offsets_dev(lm_engine* e, const uint8_t* d_levels, int n0, int n1, int n2, int n_levels, int alpha,
                             const int8_t* offsets, int n_offsets, int64_t* dependence, int64_t* ngtdm_counts,
                             int64_t* ngtdm_sums, void* stream) {
  static const char* fn = "lm_neighbour_offsets_dev";
  if (!e || !d_levels || !dependence || !ngtdm_counts || !ngtdm_sums) return fail(-1, "%s: NULL argument", fn);
  RC(check_offsets(fn, offsets, n_offsets));
  RC(check_texture_volume(fn, n0, n1, n2));
  if (n_levels < 1 || n_levels > kTextureMaxLevels) return fail(-1, "%s: n_levels %d not in [1,%d]", fn, n_levels, kTextureMaxLevels);
  if (alpha < 0) return fail(-1, "%s: alpha %d is negative", fn, alpha);
  RC(analysis_inputs(e, fn, stream, {{"d_levels", d_levels}}));
  const int rc = neighbour_offsets(e->texture, d_levels, n0, n1, n2, n_levels, alpha, offsets, n_offsets, dependence,
                                   ngtdm_counts, ngtdm_sums, e->num_sms, e->st, &e->launches);
  if (rc) return texture_device_error(fn, rc, n_levels);
  return 0;
}

int lm_zone_sizes_plane_dev(lm_engine* e, const uint8_t* d_levels, int n0, int n1, int n2, int axis, int64_t* n_pairs,
                            int64_t* sizes, int64_t* counts, size_t max_pairs, void* stream) {
  static const char* fn = "lm_zone_sizes_plane_dev";
  if (!e || !d_levels || !n_pairs || !sizes || !counts) return fail(-1, "%s: NULL argument", fn);
  if (axis < 0 || axis > 2) return fail(-1, "%s: axis %d not in [0,2]", fn, axis);
  RC(check_texture_volume(fn, n0, n1, n2));
  const size_t n = (size_t)n0 * n1 * n2;
  if (max_pairs < laa_max_pairs(n))
    return fail(-1, "%s: max_pairs %zu below lm_laa_max_pairs(%zu) = %zu", fn, max_pairs, n, laa_max_pairs(n));
  RC(analysis_inputs(e, fn, stream, {{"d_levels", d_levels}}));
  RC(zone_sizes_plane(e->clusters, d_levels, n0, n1, n2, axis, n_pairs, sizes, counts, max_pairs, e->num_sms, e->st,
                      &e->launches));
  return 0;
}

// The argument checks the two shape calls share: the shape (fewer than 2^32 voxels, every axis below 2^30).
static int check_shape_volume(const char* fn, int n0, int n1, int n2) {
  if (n0 < 1 || n1 < 1 || n2 < 1) return fail(-1, "%s: empty volume (%d,%d,%d)", fn, n0, n1, n2);
  const size_t n = (size_t)n0 * n1 * n2;
  if (n >= ((size_t)1 << 32)) return fail(-1, "%s: %zu voxels, the shape calls take fewer than 2^32", fn, n);
  if (n0 >= (1 << 30) || n1 >= (1 << 30) || n2 >= (1 << 30)) return fail(-1, "%s: (%d,%d,%d): an axis of 2^30 or more", fn, n0, n1, n2);
  return 0;
}

int lm_shape_sums_dev(lm_engine* e, const uint8_t* d_mask, int n0, int n1, int n2, int64_t* cube_counts, int64_t* cube_possum,
                      int64_t* moments, void* stream) {
  static const char* fn = "lm_shape_sums_dev";
  if (!e || !d_mask || !cube_counts || !cube_possum || !moments) return fail(-1, "%s: NULL argument", fn);
  RC(check_shape_volume(fn, n0, n1, n2));
  RC(analysis_inputs(e, fn, stream, {{"d_mask", d_mask}}));
  RC(shape_sums(e->shape, d_mask, n0, n1, n2, cube_counts, cube_possum, moments, e->num_sms, e->st, &e->launches));
  return 0;
}

int lm_max_diameters_dev(lm_engine* e, const uint8_t* d_mask, int n0, int n1, int n2, int row, const double* spacing, double* d2,
                         void* stream) {
  static const char* fn = "lm_max_diameters_dev";
  if (!e || !d_mask || !spacing || !d2) return fail(-1, "%s: NULL argument", fn);
  RC(check_shape_volume(fn, n0, n1, n2));
  if (row < 1 || row > 256) return fail(-1, "%s: row %d not in [1,256]", fn, row);
  for (int k = 0; k < 3; ++k)
    if (!(spacing[k] > 0.0 && spacing[k] < INFINITY)) return fail(-1, "%s: spacing[%d] = %g is not finite and positive", fn, k, spacing[k]);
  RC(analysis_inputs(e, fn, stream, {{"d_mask", d_mask}}));
  RC(max_diameters(e->shape, d_mask, n0, n1, n2, row, spacing, d2, e->num_sms, e->st, &e->launches));
  return 0;
}

// The arguments the two mesh calls share: the shape and row as the shape calls, and the triangle table (see
// lm_mesh_counts_dev): offsets non-decreasing from 0, at most kMeshMaxTriangles per configuration, and every code an edge
// from corner a along axis m that crosses in its configuration.
static int check_mesh_args(const char* fn, int n0, int n1, int n2, int row, const int32_t* off, const uint8_t* codes) {
  RC(check_shape_volume(fn, n0, n1, n2));
  if (row < 1 || row > 256) return fail(-1, "%s: row %d not in [1,256]", fn, row);
  if (off[0] != 0) return fail(-1, "%s: tri_offsets[0] = %d, expected 0", fn, off[0]);
  for (int c = 0; c < kMeshConfigs; ++c) {
    const int nt = off[c + 1] - off[c];
    if (nt < 0 || nt > kMeshMaxTriangles)
      return fail(-1, "%s: configuration %d has %d triangles, the table allows 0..%d", fn, c, nt, kMeshMaxTriangles);
    if ((c == 0 || c == kMeshConfigs - 1) && nt) return fail(-1, "%s: configuration %d cannot have triangles", fn, c);
    for (int i = 3 * off[c]; i < 3 * off[c + 1]; ++i) {
      const int a = codes[i] >> 2, m = codes[i] & 3;
      if (a > 7 || m > 2 || (a & (4 >> m)))
        return fail(-1, "%s: configuration %d: code %d is not an edge (corner << 2 | axis)", fn, c, codes[i]);
      if (((c >> a) & 1) == ((c >> (a | (4 >> m))) & 1))
        return fail(-1, "%s: configuration %d: the edge of code %d does not cross", fn, c, codes[i]);
    }
  }
  return 0;
}

int lm_mesh_counts_dev(lm_engine* e, const uint8_t* d_mask, int n0, int n1, int n2, int row, const int32_t* tri_offsets,
                       const uint8_t* tri_codes, int64_t* n_vertices, int64_t* n_triangles, void* stream) {
  static const char* fn = "lm_mesh_counts_dev";
  if (!e || !d_mask || !tri_offsets || !tri_codes || !n_vertices || !n_triangles) return fail(-1, "%s: NULL argument", fn);
  RC(check_mesh_args(fn, n0, n1, n2, row, tri_offsets, tri_codes));
  RC(analysis_inputs(e, fn, stream, {{"d_mask", d_mask}}));
  RC(mesh_counts(e->mesh, d_mask, n0, n1, n2, row, MeshTable{tri_offsets, tri_codes}, n_vertices, n_triangles, e->num_sms,
                 e->st, &e->launches));
  return 0;
}

int lm_mesh_emit_dev(lm_engine* e, const uint8_t* d_mask, int n0, int n1, int n2, int row, const int32_t* tri_offsets,
                     const uint8_t* tri_codes, const double* geometry, int flags, int64_t n_vertices, int64_t n_triangles,
                     int32_t* d_index2, double* d_vertices, int32_t* d_triangles, void* stream) {
  static const char* fn = "lm_mesh_emit_dev";
  if (!e || !d_mask || !tri_offsets || !tri_codes || !geometry) return fail(-1, "%s: NULL argument", fn);
  RC(check_mesh_args(fn, n0, n1, n2, row, tri_offsets, tri_codes));
  if (flags & ~LM_MESH_RAS) return fail(-1, "%s: unknown flags 0x%x", fn, flags);
  if (n_vertices < 0 || n_vertices > INT32_MAX || n_triangles < 0 || n_triangles > INT32_MAX)
    return fail(-1, "%s: %lld vertices / %lld triangles, int32 indices take at most 2^31 - 1", fn, (long long)n_vertices,
                (long long)n_triangles);
  if ((n_vertices && (!d_index2 || !d_vertices)) || (n_triangles && !d_triangles)) return fail(-1, "%s: NULL output", fn);
  MeshPlacement P{};
  for (int k = 0; k < 15; ++k)
    if (!isfinite(geometry[k])) return fail(-1, "%s: geometry[%d] = %g is not finite", fn, k, geometry[k]);
  for (int k = 0; k < 3; ++k) {
    P.o[k] = geometry[k];
    P.s[k] = geometry[12 + k];
    if (!(P.s[k] > 0.0)) return fail(-1, "%s: spacing %g along %c is not positive", fn, P.s[k], "xyz"[k]);
  }
  for (int k = 0; k < 9; ++k) P.d[k] = geometry[3 + k];
  const double* D = P.d;
  const double det = D[0] * (D[4] * D[8] - D[5] * D[7]) - D[1] * (D[3] * D[8] - D[5] * D[6]) + D[2] * (D[3] * D[7] - D[4] * D[6]);
  if (det == 0.0) return fail(-1, "%s: the direction matrix is singular", fn);
  P.ras = flags & LM_MESH_RAS;
  P.reverse = det < 0.0;
  const size_t nv = (size_t)n_vertices, nt = (size_t)n_triangles;
  RC(analysis_inputs(e, fn, stream, {{"d_mask", d_mask}, {"d_index2", nv ? d_index2 : nullptr},
                                     {"d_vertices", nv ? d_vertices : nullptr}, {"d_triangles", nt ? d_triangles : nullptr}}));
  const int rc = mesh_emit(e->mesh, d_mask, n0, n1, n2, row, MeshTable{tri_offsets, tri_codes}, P, n_vertices, n_triangles,
                           d_index2, d_vertices, d_triangles, e->num_sms, e->st, &e->launches);
  if (rc == -2) return fail(-1, "%s: n_vertices / n_triangles (%lld / %lld) are not the row's counts", fn,
                            (long long)n_vertices, (long long)n_triangles);
  return rc;
}

// The row arguments the two first-order calls share: modes, the band and the exact rows' base; `pass` 0 (sums) also
// checks the levels, 1 (splits) the split points and the float rows' centres.
static int check_first_order_rows(const char* fn, int dtype, const FirstOrderRows& r, int pass) {
  const bool int_dtype = dtype == LM_DTYPE_U8 || dtype == LM_DTYPE_I8 || dtype == LM_DTYPE_I16 || dtype == LM_DTYPE_I32 ||
                         dtype == LM_DTYPE_I64;
  if (r.mode[0] != kFoSkip) return fail(-1, "%s: row 0 (background) has mode %d, it is never a row", fn, r.mode[0]);
  bool labels = false;
  for (int i = 1; i < kFoRows; ++i) {
    const int m = r.mode[i];
    if (m != kFoSkip && m != kFoFloat && m != kFoExact) return fail(-1, "%s: row %d: mode %d is not 0, 1 or 2", fn, i, m);
    if (m == kFoSkip) continue;
    labels |= i < 256;
    if (m == kFoExact && !int_dtype) return fail(-1, "%s: row %d: the exact mode needs an integer volume (dtype %d)", fn, i, dtype);
    if (!(r.band_lo[i] <= r.band_hi[i])) return fail(-1, "%s: row %d: band [%g, %g] is empty or NaN", fn, i, r.band_lo[i], r.band_hi[i]);
    if (m == kFoExact && (r.base[i] < -((int64_t)1 << 53) || r.base[i] > ((int64_t)1 << 53)))
      return fail(-1, "%s: row %d: base %lld beyond 2^53", fn, i, (long long)r.base[i]);
    if (m == kFoFloat && !isfinite(r.centre[i])) return fail(-1, "%s: row %d: centre %g is not finite", fn, i, r.centre[i]);
    if (pass == 0 && (r.n_levels[i] < 1 || r.n_levels[i] > kTextureMaxLevels))
      return fail(-1, "%s: row %d: n_levels %d not in [1,%d]", fn, i, r.n_levels[i], kTextureMaxLevels);
    if (pass == 1 && m == kFoExact) {
      if (r.split[i] < 0 || r.split[i] >= kFoExactSpan || r.split_band[i] < 0 || r.split_band[i] >= kFoExactSpan)
        return fail(-1, "%s: row %d: split %lld / %lld not in [0,2^20)", fn, i, (long long)r.split[i], (long long)r.split_band[i]);
    }
    if (pass == 1 && m == kFoFloat && !isfinite(r.centre_band[i]))
      return fail(-1, "%s: row %d: centre_band %g is not finite", fn, i, r.centre_band[i]);
  }
  if (labels && r.mode[256] == kFoSkip) return fail(-1, "%s: a label row needs the union row 256", fn);
  return 0;
}

static int first_order_device_error(const char* fn, int rc) {
  if (rc == kFoRange) return fail(rc, "%s: a value outside its row's exact span or level range", fn);
  return rc;
}

int lm_first_order_sums_dev(lm_engine* e, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2,
                            int bin_width, const int* mode, const int64_t* low, const int* n_levels, const int64_t* base,
                            const double* centre, const double* band_lo, const double* band_hi, int64_t* histogram,
                            uint64_t* int_sums, int64_t* band_count, double* float_sums, void* stream) {
  static const char* fn = "lm_first_order_sums_dev";
  if (!e || !d_vol || !d_mask || !mode || !low || !n_levels || !base || !centre || !band_lo || !band_hi || !histogram ||
      !int_sums || !band_count || !float_sums)
    return fail(-1, "%s: NULL argument", fn);
  RC(check_texture_volume(fn, n0, n1, n2));
  if (dtype < LM_DTYPE_I16 || dtype > LM_DTYPE_BF16) return fail(-1, "%s: unknown dtype code %d", fn, dtype);
  if (bin_width < 1) return fail(-1, "%s: bin_width %d is not positive", fn, bin_width);
  const FirstOrderRows rows{mode, low, n_levels, base, centre, nullptr, band_lo, band_hi, nullptr, nullptr};
  RC(check_first_order_rows(fn, dtype, rows, 0));
  RC(analysis_inputs(e, fn, stream, {{"d_vol", d_vol}, {"d_mask", d_mask}}));
  const int rc = first_order_sums(e->first_order, d_vol, dtype, d_mask, (size_t)n0 * n1 * n2, bin_width, rows, histogram,
                                  int_sums, band_count, float_sums, e->num_sms, e->st, &e->launches);
  if (rc) return first_order_device_error(fn, rc);
  return 0;
}

int lm_first_order_splits_dev(lm_engine* e, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2,
                              const int* mode, const int64_t* base, const int64_t* split, const int64_t* split_band,
                              const double* centre, const double* centre_band, const double* band_lo,
                              const double* band_hi, int64_t* below, double* abs_dev, void* stream) {
  static const char* fn = "lm_first_order_splits_dev";
  if (!e || !d_vol || !d_mask || !mode || !base || !split || !split_band || !centre || !centre_band || !band_lo ||
      !band_hi || !below || !abs_dev)
    return fail(-1, "%s: NULL argument", fn);
  RC(check_texture_volume(fn, n0, n1, n2));
  if (dtype < LM_DTYPE_I16 || dtype > LM_DTYPE_BF16) return fail(-1, "%s: unknown dtype code %d", fn, dtype);
  const FirstOrderRows rows{mode, nullptr, nullptr, base, centre, centre_band, band_lo, band_hi, split, split_band};
  RC(check_first_order_rows(fn, dtype, rows, 1));
  RC(analysis_inputs(e, fn, stream, {{"d_vol", d_vol}, {"d_mask", d_mask}}));
  const int rc = first_order_splits(e->first_order, d_vol, dtype, d_mask, (size_t)n0 * n1 * n2, rows, below, abs_dev,
                                    e->num_sms, e->st, &e->launches);
  if (rc) return first_order_device_error(fn, rc);
  return 0;
}

int lm_wavelet_dev(lm_engine* e, const void* d_vol, int dtype, int n0, int n1, int n2, int wavelet, int band, double* d_out,
                   void* stream) {
  static const char* fn = "lm_wavelet_dev";
  if (!e || !d_vol || !d_out) return fail(-1, "%s: NULL argument", fn);
  if (n0 < 1 || n1 < 1 || n2 < 1) return fail(-1, "%s: empty volume (%d,%d,%d)", fn, n0, n1, n2);
  const size_t n = (size_t)n0 * n1 * n2;
  if (n >= ((size_t)1 << 32)) return fail(-1, "%s: %zu voxels, the wavelet call takes fewer than 2^32", fn, n);
  if (dtype < LM_DTYPE_I16 || dtype > LM_DTYPE_BF16) return fail(-1, "%s: unknown dtype code %d", fn, dtype);
  const int taps = wavelet_taps(wavelet);
  if (!taps) return fail(-1, "%s: unknown wavelet code %d", fn, wavelet);
  if (band < 0 || band >= kWaveletBands) return fail(-1, "%s: band %d not in [0,%d)", fn, band, kWaveletBands);
  const int dims[3] = {n0, n1, n2};
  for (int a = 0; a < 3; ++a)
    if (dims[a] + (dims[a] & 1) < taps)
      return fail(-1, "%s: axis %d has %d voxels (padded %d), the filter needs at least %d", fn, a, dims[a],
                  dims[a] + (dims[a] & 1), taps);
  const uintptr_t v0 = reinterpret_cast<uintptr_t>(d_vol), o0 = reinterpret_cast<uintptr_t>(d_out);
  if (v0 < o0 + n * sizeof(double) && o0 < v0 + n * dtype_bytes(dtype)) return fail(-1, "%s: d_out overlaps d_vol", fn);
  RC(analysis_inputs(e, fn, stream, {{"d_vol", d_vol}, {"d_out", d_out}}));
  const int rc = wavelet_band(e->wavelet, d_vol, dtype, n0, n1, n2, wavelet, band, d_out, e->st, &e->launches);
  if (rc == LM_ERR_NONFINITE) return fail(rc, "%s: the volume holds a NaN or +-inf", fn);
  return rc;
}

// The volume arguments shared by the filter calls: the engine, the volume pointer, its extents and dtype code.
static int filter_volume_args(const char* fn, lm_engine* e, const void* d_vol, int dtype, int n0, int n1, int n2) {
  if (!e || !d_vol) return fail(-1, "%s: NULL argument", fn);
  if (n0 < 1 || n1 < 1 || n2 < 1) return fail(-1, "%s: empty volume (%d,%d,%d)", fn, n0, n1, n2);
  const size_t n = (size_t)n0 * n1 * n2;
  if (n >= ((size_t)1 << 32)) return fail(-1, "%s: %zu voxels, the filter calls take fewer than 2^32", fn, n);
  if (dtype < LM_DTYPE_I16 || dtype > LM_DTYPE_BF16) return fail(-1, "%s: unknown dtype code %d", fn, dtype);
  return 0;
}

static bool overlaps(const void* a, size_t a_bytes, const void* b, size_t b_bytes) {
  const uintptr_t a0 = reinterpret_cast<uintptr_t>(a), b0 = reinterpret_cast<uintptr_t>(b);
  return a0 < b0 + b_bytes && b0 < a0 + a_bytes;
}

static int filter_result(const char* fn, int rc) {
  if (rc == LM_ERR_NONFINITE) return fail(rc, "%s: the volume holds a NaN or +-inf", fn);
  if (rc == LM_ERR_TABLE_RANGE) return fail(rc, "%s: a voxel lies outside the table", fn);
  return rc;
}

int lm_image_range_dev(lm_engine* e, const void* d_vol, int dtype, int n0, int n1, int n2, double* out, void* stream) {
  static const char* fn = "lm_image_range_dev";
  RC(filter_volume_args(fn, e, d_vol, dtype, n0, n1, n2));
  if (!out) return fail(-1, "%s: NULL argument", fn);
  RC(analysis_inputs(e, fn, stream, {{"d_vol", d_vol}}));
  return filter_result(fn, image_range(e->filters, d_vol, dtype, (size_t)n0 * n1 * n2, out, e->num_sms, e->st,
                                       &e->launches));
}

int lm_image_filter_dev(lm_engine* e, const void* d_vol, int dtype, int n0, int n1, int n2, int type, const double* params,
                        const double* d_table, int64_t table_min, int64_t table_len, double* d_out, void* stream) {
  static const char* fn = "lm_image_filter_dev";
  RC(filter_volume_args(fn, e, d_vol, dtype, n0, n1, n2));
  if (!d_out) return fail(-1, "%s: NULL argument", fn);
  if (type < LM_FILTER_SQUARE || type > LM_FILTER_EXPONENTIAL) return fail(-1, "%s: unknown image type code %d", fn, type);
  const size_t n = (size_t)n0 * n1 * n2;
  if (overlaps(d_vol, n * dtype_bytes(dtype), d_out, n * sizeof(double))) return fail(-1, "%s: d_out overlaps d_vol", fn);
  double param = 0.0;
  if (d_table) {
    const bool integer = dtype == LM_DTYPE_U8 || dtype == LM_DTYPE_I8 || dtype == LM_DTYPE_I16 || dtype == LM_DTYPE_I32 ||
                         dtype == LM_DTYPE_I64;
    if (!integer) return fail(-1, "%s: a table needs an integer volume, got dtype code %d", fn, dtype);
    if (table_len < 1 || table_len > ((int64_t)1 << 20))
      return fail(-1, "%s: table length %lld not in [1, 2^20]", fn, (long long)table_len);
    if (table_min > INT64_MAX - table_len) return fail(-1, "%s: table [%lld, +%lld) overflows int64", fn,
                                                       (long long)table_min, (long long)table_len);
    if (overlaps(d_table, (size_t)table_len * sizeof(double), d_out, n * sizeof(double)))
      return fail(-1, "%s: d_out overlaps d_table", fn);
  } else {
    if (!params) return fail(-1, "%s: NULL params without a table", fn);
    param = params[0];
    if (!isfinite(param)) return fail(-1, "%s: params[0] = %g is not finite", fn, param);
  }
  RC(analysis_inputs(e, fn, stream, {{"d_vol", d_vol}, {"d_out", d_out}, {"d_table", d_table}}));
  return filter_result(fn, image_filter(e->filters, d_vol, dtype, n, type, param, d_table, table_min, table_len, d_out,
                                        e->num_sms, e->st, &e->launches));
}

int lm_gradient_dev(lm_engine* e, const void* d_vol, int dtype, int n0, int n1, int n2, const double* spacing_xyz,
                    double* d_out, void* stream) {
  static const char* fn = "lm_gradient_dev";
  RC(filter_volume_args(fn, e, d_vol, dtype, n0, n1, n2));
  if (!d_out || !spacing_xyz) return fail(-1, "%s: NULL argument", fn);
  double inv[3];
  for (int a = 0; a < 3; ++a) {
    if (!(isfinite(spacing_xyz[a]) && spacing_xyz[a] > 0.0))
      return fail(-1, "%s: spacing %g along %c is not a finite positive size", fn, spacing_xyz[a], "xyz"[a]);
    inv[a] = 1.0 / spacing_xyz[a];
  }
  const size_t n = (size_t)n0 * n1 * n2;
  if (overlaps(d_vol, n * dtype_bytes(dtype), d_out, n * sizeof(double))) return fail(-1, "%s: d_out overlaps d_vol", fn);
  RC(analysis_inputs(e, fn, stream, {{"d_vol", d_vol}, {"d_out", d_out}}));
  return filter_result(fn, gradient_magnitude(e->filters, d_vol, dtype, n0, n1, n2, inv, d_out, e->st, &e->launches));
}

int lm_bspline_coefficients_dev(lm_engine* e, const void* d_vol, int dtype, int n0, int n1, int n2, double* d_coeff,
                                void* stream) {
  static const char* fn = "lm_bspline_coefficients_dev";
  RC(filter_volume_args(fn, e, d_vol, dtype, n0, n1, n2));
  if (!d_coeff) return fail(-1, "%s: NULL argument", fn);
  const size_t n = (size_t)n0 * n1 * n2;
  if (overlaps(d_vol, n * dtype_bytes(dtype), d_coeff, n * sizeof(double)))
    return fail(-1, "%s: d_coeff overlaps d_vol", fn);
  RC(analysis_inputs(e, fn, stream, {{"d_vol", d_vol}, {"d_coeff", d_coeff}}));
  return filter_result(fn, bspline_coefficients(e->resample, d_vol, dtype, n0, n1, n2, d_coeff, e->st, &e->launches));
}

int lm_resample_dev(lm_engine* e, const void* d_vol, int dtype, const double* d_coeff, const uint8_t* d_mask, int n0, int n1,
                    int n2, const double* d_cz, const double* d_cy, const double* d_cx, int m0, int m1, int m2,
                    int interpolator, void* d_out, uint8_t* d_out_mask, void* stream) {
  static const char* fn = "lm_resample_dev";
  RC(filter_volume_args(fn, e, d_vol, dtype, n0, n1, n2));
  if (!d_mask || !d_cz || !d_cy || !d_cx || !d_out || !d_out_mask) return fail(-1, "%s: NULL argument", fn);
  if (interpolator != LM_RESAMPLE_BSPLINE && interpolator != LM_RESAMPLE_NEAREST)
    return fail(-1, "%s: unknown interpolator code %d", fn, interpolator);
  if (interpolator == LM_RESAMPLE_BSPLINE && !d_coeff) return fail(-1, "%s: NULL d_coeff for the B-spline", fn);
  if (m0 < 1 || m1 < 1 || m2 < 1) return fail(-1, "%s: empty output grid (%d,%d,%d)", fn, m0, m1, m2);
  const size_t n = (size_t)n0 * n1 * n2, m = (size_t)m0 * m1 * m2;
  if (m >= ((size_t)1 << 32)) return fail(-1, "%s: %zu output voxels, the call takes fewer than 2^32", fn, m);
  const size_t out_bytes = m * dtype_bytes(dtype);
  const struct { const char* name; const void* p; size_t bytes; } ins[] = {
      {"d_vol", d_vol, n * dtype_bytes(dtype)},
      {"d_coeff", interpolator == LM_RESAMPLE_BSPLINE ? d_coeff : nullptr, n * sizeof(double)},
      {"d_mask", d_mask, n},
      {"d_cz", d_cz, (size_t)m0 * sizeof(double)},
      {"d_cy", d_cy, (size_t)m1 * sizeof(double)},
      {"d_cx", d_cx, (size_t)m2 * sizeof(double)}};
  for (const auto& a : ins) {
    if (!a.p) continue;
    if (overlaps(a.p, a.bytes, d_out, out_bytes)) return fail(-1, "%s: d_out overlaps %s", fn, a.name);
    if (overlaps(a.p, a.bytes, d_out_mask, m)) return fail(-1, "%s: d_out_mask overlaps %s", fn, a.name);
  }
  if (overlaps(d_out, out_bytes, d_out_mask, m)) return fail(-1, "%s: d_out_mask overlaps d_out", fn);
  RC(analysis_inputs(e, fn, stream, {{"d_vol", d_vol}, {"d_coeff", ins[1].p}, {"d_mask", d_mask}, {"d_cz", d_cz},
                                     {"d_cy", d_cy}, {"d_cx", d_cx}, {"d_out", d_out}, {"d_out_mask", d_out_mask}}));
  // the tables are checked on the host: the engine's stream has waited for the caller's, so they are complete
  std::vector<double> tab((size_t)m0 + m1 + m2);
  CU(cudaMemcpyAsync(tab.data(), d_cz, (size_t)m0 * sizeof(double), cudaMemcpyDeviceToHost, e->st));
  CU(cudaMemcpyAsync(tab.data() + m0, d_cy, (size_t)m1 * sizeof(double), cudaMemcpyDeviceToHost, e->st));
  CU(cudaMemcpyAsync(tab.data() + m0 + m1, d_cx, (size_t)m2 * sizeof(double), cudaMemcpyDeviceToHost, e->st));
  CU(cudaStreamSynchronize(e->st));
  for (size_t k = 0; k < tab.size(); ++k)
    if (!isfinite(tab[k])) {
      const char* t = k < (size_t)m0 ? "d_cz" : (k < (size_t)m0 + m1 ? "d_cy" : "d_cx");
      return fail(-1, "%s: %s holds a NaN or +-inf", fn, t);
    }
  const int rc = resample_volume(e->resample, d_vol, dtype, d_coeff, d_mask, n0, n1, n2, d_cz, d_cy, d_cx, m0, m1, m2,
                                 interpolator, d_out, d_out_mask, e->st, &e->launches);
  if (rc == LM_ERR_NONFINITE) return fail(rc, "%s: a sampled value is a NaN or +-inf", fn);
  return rc;
}

int lm_laplacian_of_gaussian_dev(lm_engine* e, const void* d_vol, int dtype, int n0, int n1, int n2,
                                 const double* spacing_xyz, double sigma_mm, double* d_work0, double* d_work1,
                                 double* d_out, void* stream) {
  static const char* fn = "lm_laplacian_of_gaussian_dev";
  RC(filter_volume_args(fn, e, d_vol, dtype, n0, n1, n2));
  if (!spacing_xyz || !d_work0 || !d_work1 || !d_out) return fail(-1, "%s: NULL argument", fn);
  if (n0 < 4 || n1 < 4 || n2 < 4) return fail(-1, "%s: extents (%d,%d,%d), every axis needs 4 voxels", fn, n0, n1, n2);
  if (!(isfinite(sigma_mm) && sigma_mm > 0.0)) return fail(-1, "%s: sigma %g is not a finite size > 0 mm", fn, sigma_mm);
  const int extent[3] = {n2, n1, n0};   // x, y, z
  LogLine smooth[3], deriv[3];
  for (int a = 0; a < 3; ++a) {
    if (!(isfinite(spacing_xyz[a]) && spacing_xyz[a] > 0.0))
      return fail(-1, "%s: spacing %g along %c is not a finite positive size", fn, spacing_xyz[a], "xyz"[a]);
    const double sd = sigma_mm / spacing_xyz[a];
    if ((double)extent[a] < ceil(sd) + 1.0)
      return fail(-1, "%s: sigma %g mm needs at least ceil(sigma / spacing) + 1 = %.0f voxels along %c, the volume has %d",
                  fn, sigma_mm, ceil(sd) + 1.0, "xyz"[a], extent[a]);
    smooth[a] = log_line_coefficients(sd, 0);
    deriv[a] = log_line_coefficients(sd, 2);
  }
  const size_t n = (size_t)n0 * n1 * n2, f64 = n * sizeof(double);
  const struct { const char* name; const void* p; size_t bytes; } bufs[] = {
      {"d_vol", d_vol, n * dtype_bytes(dtype)}, {"d_work0", d_work0, f64}, {"d_work1", d_work1, f64}, {"d_out", d_out, f64}};
  for (int i = 1; i < 4; ++i)
    for (int j = 0; j < i; ++j)
      if (overlaps(bufs[i].p, bufs[i].bytes, bufs[j].p, bufs[j].bytes))
        return fail(-1, "%s: %s overlaps %s", fn, bufs[i].name, bufs[j].name);
  RC(analysis_inputs(e, fn, stream, {{"d_vol", d_vol}, {"d_work0", d_work0}, {"d_work1", d_work1}, {"d_out", d_out}}));
  return filter_result(fn, laplacian_of_gaussian(e->laplacian, d_vol, dtype, n0, n1, n2, smooth, deriv, d_work0, d_work1, d_out,
                                                 e->st, &e->launches));
}

int lm_first_order_maps_dev(lm_engine* e, const void* d_vol, int dtype, const uint8_t* d_mask, int n0, int n1, int n2,
                            int row, int radius, int masked, int bin_width, int64_t low, int n_levels, int mode,
                            int64_t base, int64_t shift, double voxel_volume, double init_value, uint32_t feature_bits,
                            const double* d_entropy_table, int64_t table_len, double* d_out, void* stream) {
  static const char* fn = "lm_first_order_maps_dev";
  if (!e || !d_vol || !d_mask || !d_entropy_table || !d_out) return fail(-1, "%s: NULL argument", fn);
  RC(check_texture_volume(fn, n0, n1, n2));
  if (dtype < LM_DTYPE_I16 || dtype > LM_DTYPE_BF16) return fail(-1, "%s: unknown dtype code %d", fn, dtype);
  if (row < 1 || row > 256) return fail(-1, "%s: row %d not in [1,256]", fn, row);
  if (radius < 1 || radius > kFomMaxRadius) return fail(-1, "%s: radius %d not in [1,%d]", fn, radius, kFomMaxRadius);
  if (masked != 0 && masked != 1) return fail(-1, "%s: masked %d is not 0 or 1", fn, masked);
  if (bin_width < 1) return fail(-1, "%s: bin_width %d is not positive", fn, bin_width);
  if (n_levels < 1 || n_levels > kTextureMaxLevels) return fail(-1, "%s: n_levels %d not in [1,%d]", fn, n_levels, kTextureMaxLevels);
  const bool integer = dtype == LM_DTYPE_U8 || dtype == LM_DTYPE_I8 || dtype == LM_DTYPE_I16 || dtype == LM_DTYPE_I32 ||
                       dtype == LM_DTYPE_I64;
  if (mode != LM_FOM_FLOAT && mode != LM_FOM_EXACT) return fail(-1, "%s: mode %d is not LM_FOM_FLOAT or LM_FOM_EXACT", fn, mode);
  if (mode == LM_FOM_EXACT && !integer) return fail(-1, "%s: the exact mode needs an integer volume (dtype %d)", fn, dtype);
  const int64_t lim53 = (int64_t)1 << 53, lim58 = (int64_t)1 << 58, lim62 = (int64_t)1 << 62;
  if (mode == LM_FOM_EXACT && (base < -lim53 || base > lim53)) return fail(-1, "%s: base %lld beyond 2^53", fn, (long long)base);
  if (low <= -lim62 || low >= lim62) return fail(-1, "%s: low %lld beyond 2^62", fn, (long long)low);
  if (shift <= -lim58 || shift >= lim58 || (mode == LM_FOM_EXACT && (base + shift <= -lim58 || base + shift >= lim58)))
    return fail(-1, "%s: shift %lld: |shift| and |base + shift| must stay below 2^58", fn, (long long)shift);
  if (!(isnan(voxel_volume) || (isfinite(voxel_volume) && voxel_volume > 0.0)))
    return fail(-1, "%s: voxel_volume %g is neither NaN nor finite and positive", fn, voxel_volume);
  if (feature_bits == 0 || (feature_bits >> kFomFeatures))
    return fail(-1, "%s: feature_bits 0x%x: set one or more of the %d feature bits and no other", fn, feature_bits, kFomFeatures);
  const int64_t K = (int64_t)(2 * radius + 1) * (2 * radius + 1) * (2 * radius + 1);
  if (table_len != K * (K + 1) / 2)
    return fail(-1, "%s: table_len %lld, radius %d needs %lld", fn, (long long)table_len, radius, (long long)(K * (K + 1) / 2));
  const size_t n = (size_t)n0 * n1 * n2, out_bytes = (size_t)__builtin_popcount(feature_bits) * n * sizeof(double);
  if (overlaps(d_vol, n * dtype_bytes(dtype), d_out, out_bytes)) return fail(-1, "%s: d_out overlaps d_vol", fn);
  if (overlaps(d_mask, n, d_out, out_bytes)) return fail(-1, "%s: d_out overlaps d_mask", fn);
  if (overlaps(d_entropy_table, (size_t)table_len * sizeof(double), d_out, out_bytes))
    return fail(-1, "%s: d_out overlaps d_entropy_table", fn);
  RC(analysis_inputs(e, fn, stream, {{"d_vol", d_vol}, {"d_mask", d_mask}, {"d_entropy_table", d_entropy_table},
                                     {"d_out", d_out}}));
  const FomArgs a{row, radius, masked, bin_width, n_levels, mode == LM_FOM_EXACT, (long long)low, (long long)base,
                  (long long)shift, voxel_volume, init_value, feature_bits, d_entropy_table};
  const int rc = first_order_maps(e->fo_maps, d_vol, dtype, d_mask, n0, n1, n2, a, d_out, e->num_sms, e->st, &e->launches);
  if (rc == LM_ERR_NONFINITE) return fail(rc, "%s: a window holds a +-inf value", fn);
  if (rc == kFomRange) return fail(rc, "%s: a value outside the exact span or a level outside 1..%d", fn, n_levels);
  return rc;
}

int lm_glcm_maps_dev(lm_engine* e, const uint8_t* d_levels, const uint8_t* d_mask, int n0, int n1, int n2, int row,
                     int radius, int n_levels, double init_value, uint32_t feature_bits, const double* d_entropy_table,
                     int64_t table_len, double* d_out, void* stream) {
  static const char* fn = "lm_glcm_maps_dev";
  if (!e || !d_levels || !d_mask || !d_entropy_table || !d_out) return fail(-1, "%s: NULL argument", fn);
  RC(check_texture_volume(fn, n0, n1, n2));
  if (row < 1 || row > 256) return fail(-1, "%s: row %d not in [1,256]", fn, row);
  if (radius < 1 || radius > kGlcmMapsMaxRadius) return fail(-1, "%s: radius %d not in [1,%d]", fn, radius, kGlcmMapsMaxRadius);
  if (n_levels < 1 || n_levels > kTextureMaxLevels) return fail(-1, "%s: n_levels %d not in [1,%d]", fn, n_levels, kTextureMaxLevels);
  if (feature_bits == 0 || (feature_bits >> kGlcmMapsFeatures))
    return fail(-1, "%s: feature_bits 0x%x: set one or more of the %d feature bits and no other", fn, feature_bits,
                kGlcmMapsFeatures);
  const int64_t nmax = glcm_maps_max_n(radius);
  if (table_len != nmax * (nmax + 1) / 2)
    return fail(-1, "%s: table_len %lld, radius %d needs %lld", fn, (long long)table_len, radius, (long long)(nmax * (nmax + 1) / 2));
  const size_t n = (size_t)n0 * n1 * n2, out_bytes = (size_t)__builtin_popcount(feature_bits) * n * sizeof(double);
  if (overlaps(d_levels, n, d_out, out_bytes)) return fail(-1, "%s: d_out overlaps d_levels", fn);
  if (overlaps(d_mask, n, d_out, out_bytes)) return fail(-1, "%s: d_out overlaps d_mask", fn);
  if (overlaps(d_entropy_table, (size_t)table_len * sizeof(double), d_out, out_bytes))
    return fail(-1, "%s: d_out overlaps d_entropy_table", fn);
  RC(analysis_inputs(e, fn, stream, {{"d_levels", d_levels}, {"d_mask", d_mask}, {"d_entropy_table", d_entropy_table},
                                     {"d_out", d_out}}));
  const GlcmMapsArgs a{row, radius, n_levels, init_value, feature_bits, d_entropy_table};
  const int rc = glcm_maps(e->glcm_maps, d_levels, d_mask, n0, n1, n2, a, d_out, e->num_sms, e->st, &e->launches);
  if (rc == kGlcmMapsRange) return fail(rc, "%s: a level above n_levels (%d) in a window", fn, n_levels);
  return rc;
}

int lm_texture_maps_dev(lm_engine* e, const uint8_t* d_levels, const uint8_t* d_mask, int n0, int n1, int n2, int row,
                        int radius, int n_levels, int cls, int alpha, double init_value, uint32_t feature_bits,
                        const double* d_entropy_table, int64_t table_len, double* d_out, void* stream) {
  static const char* fn = "lm_texture_maps_dev";
  if (!e || !d_levels || !d_mask || !d_entropy_table || !d_out) return fail(-1, "%s: NULL argument", fn);
  RC(check_texture_volume(fn, n0, n1, n2));
  if (cls < LM_TEXMAP_GLSZM || cls > LM_TEXMAP_NGTDM)
    return fail(-1, "%s: class %d is not LM_TEXMAP_GLSZM, _GLRLM, _GLDM or _NGTDM", fn, cls);
  if (row < 1 || row > 256) return fail(-1, "%s: row %d not in [1,256]", fn, row);
  if (radius < 1 || radius > kTexMapsMaxRadius) return fail(-1, "%s: radius %d not in [1,%d]", fn, radius, kTexMapsMaxRadius);
  if (n_levels < 1 || n_levels > kTextureMaxLevels) return fail(-1, "%s: n_levels %d not in [1,%d]", fn, n_levels, kTextureMaxLevels);
  if (alpha < 0) return fail(-1, "%s: alpha %d is negative", fn, alpha);
  const int nf = texture_maps_features(cls);
  if (feature_bits == 0 || (feature_bits >> nf))
    return fail(-1, "%s: feature_bits 0x%x: set one or more of the class's %d feature bits and no other", fn, feature_bits, nf);
  const int64_t K = (int64_t)(2 * radius + 1) * (2 * radius + 1) * (2 * radius + 1);
  if (table_len != K * (K + 1) / 2)
    return fail(-1, "%s: table_len %lld, radius %d needs %lld", fn, (long long)table_len, radius, (long long)(K * (K + 1) / 2));
  const size_t n = (size_t)n0 * n1 * n2, out_bytes = (size_t)__builtin_popcount(feature_bits) * n * sizeof(double);
  if (overlaps(d_levels, n, d_out, out_bytes)) return fail(-1, "%s: d_out overlaps d_levels", fn);
  if (overlaps(d_mask, n, d_out, out_bytes)) return fail(-1, "%s: d_out overlaps d_mask", fn);
  if (overlaps(d_entropy_table, (size_t)table_len * sizeof(double), d_out, out_bytes))
    return fail(-1, "%s: d_out overlaps d_entropy_table", fn);
  RC(analysis_inputs(e, fn, stream, {{"d_levels", d_levels}, {"d_mask", d_mask}, {"d_entropy_table", d_entropy_table},
                                     {"d_out", d_out}}));
  const TextureMapsArgs a{row, radius, n_levels, cls, alpha, init_value, feature_bits, d_entropy_table};
  const int rc = texture_maps(e->texture_maps, d_levels, d_mask, n0, n1, n2, a, d_out, e->num_sms, e->st, &e->launches);
  if (rc == kTexMapsRange) return fail(rc, "%s: a level above n_levels (%d) in a window", fn, n_levels);
  return rc;
}

int lm_shard_init(lm_engine* e, int rank, int world, int max_slices) {
  if (!e) return fail(-1, "lm_shard_init: NULL engine");
  if (world < 1 || world > kShardMaxWorld || rank < 0 || rank >= world) return fail(-1, "lm_shard_init: rank %d / world %d", rank, world);
  if (max_slices < 1) return fail(-1, "lm_shard_init: max_slices < 1");
  CU(cudaSetDevice(e->device));
  CU(cudaStreamSynchronize(e->st));
  shard_release(e);
  e->shard.rank = rank; e->shard.world = world;
  const size_t per = ((size_t)max_slices + world - 1) / world;
  e->shard.slice_cap = per * world;
  e->shard.block_bytes = shard_block_bytes(e->shard.slice_cap, (size_t)R * R);
  void* p = nullptr;
  CU(cudaMalloc(&p, e->shard.block_bytes));
  e->shard.block[rank] = static_cast<uint8_t*>(p);
  CU(cudaMemset(p, 0, e->shard.block_bytes));
  CU(cudaMallocHost(&e->h_shard_err, sizeof(uint32_t)));
  *e->h_shard_err = 0;
  e->shard_epoch = 0;
  e->shard_connected = (world == 1);
  return 0;
}

size_t lm_shard_handle_bytes(void) { return sizeof(cudaIpcMemHandle_t); }

int lm_shard_export(lm_engine* e, void* handle_out) {
  if (!e || !handle_out) return fail(-1, "lm_shard_export: NULL argument");
  if (!e->shard.block[e->shard.rank]) return fail(-51, "lm_shard_export: call lm_shard_init first");
  CU(cudaSetDevice(e->device));
  cudaIpcMemHandle_t h;
  CU(cudaIpcGetMemHandle(&h, e->shard.block[e->shard.rank]));
  memcpy(handle_out, &h, sizeof(h));
  return 0;
}

int lm_shard_connect(lm_engine* e, const void* handles) {
  if (!e || !handles) return fail(-1, "lm_shard_connect: NULL argument");
  if (!e->shard.block[e->shard.rank]) return fail(-51, "lm_shard_connect: call lm_shard_init first");
  CU(cudaSetDevice(e->device));
  const uint8_t* hb = static_cast<const uint8_t*>(handles);
  for (int p = 0; p < e->shard.world; ++p) {
    if (p == e->shard.rank || e->shard.block[p]) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, hb + (size_t)p * sizeof(h), sizeof(h));
    void* ptr = nullptr;
    CU(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
    e->shard.block[p] = static_cast<uint8_t*>(ptr);
  }
  e->shard_connected = true;
  return 0;
}

int lm_shard_labels(lm_engine* e, void** d_boxes, void** d_labels, size_t* slice_cap) {
  if (!e) return fail(-1, "lm_shard_labels: NULL engine");
  if (!e->shard.block[e->shard.rank]) return fail(-51, "lm_shard_labels: call lm_shard_init first");
  if (d_boxes) *d_boxes = e->shard.block[e->shard.rank] + shard_boxes_offset();
  if (d_labels) *d_labels = e->shard.block[e->shard.rank] + shard_labels_offset(e->shard.slice_cap);
  if (slice_cap) *slice_cap = e->shard.slice_cap;
  return 0;
}

int lm_apply_volume_sharded_dev(lm_engine* e, int slot, const int16_t* d_vol, int S, int H, int W, int flags, uint8_t* d_out) {
  if (!e || !d_vol || !d_out) return fail(-1, "lm_apply_volume_sharded_dev: NULL argument");
  if (S < 1 || H < 1 || W < 1) return fail(-1, "lm_apply_volume_sharded_dev: empty volume");
  if (!e->shard_connected) return fail(-51, "lm_apply_volume_sharded_dev: call lm_shard_init / lm_shard_connect first");
  if ((size_t)S > e->shard.slice_cap) return fail(-52, "lm_apply_volume_sharded_dev: %d slices exceed the gather capacity %zu", S, e->shard.slice_cap);
  CU(cudaSetDevice(e->device));
  RC(run_checked(e, [&]() -> int {
    e->launches = 0;
    e->ev_used = 0;
    CU(cudaEventRecord(e->ev[0], e->st));
    RC(sharded_dev(e, slot, d_vol, S, H, W, flags, d_out));
    CU(cudaEventRecord(e->ev[6], e->st));
    return 0;
  }));
  collect_timings(e);
  return shard_check(e);
}

int lm_apply_volume_sharded(lm_engine* e, int slot, const int16_t* vol, int S, int H, int W, int flags, uint8_t* out) {
  if (!e || !vol) return fail(-1, "lm_apply_volume_sharded: NULL argument");
  if (S < 1 || H < 1 || W < 1) return fail(-1, "lm_apply_volume_sharded: empty volume");
  if (!e->shard_connected) return fail(-51, "lm_apply_volume_sharded: call lm_shard_init / lm_shard_connect first");
  if ((size_t)S > e->shard.slice_cap) return fail(-52, "lm_apply_volume_sharded: %d slices exceed the gather capacity %zu", S, e->shard.slice_cap);
  CU(cudaSetDevice(e->device));
  const size_t n = (size_t)S * H * W, plane = (size_t)H * W;
  RC(e->d_vol.reserve(n));
  RC(e->d_out.reserve(n));
  int lo, hi;
  shard_range(S, e->shard.rank, e->shard.world, &lo, &hi);
  RC(run_checked(e, [&]() -> int {
    e->launches = 0;
    e->ev_used = 0;
    CU(cudaEventRecord(e->ev[0], e->st));
    if (hi > lo)  // only this rank's slab crosses the PCIe bus
      CU(cudaMemcpyAsync(e->d_vol.p + (size_t)lo * plane, vol + (size_t)lo * plane, (size_t)(hi - lo) * plane * sizeof(int16_t),
                         cudaMemcpyHostToDevice, e->st));
    RC(sharded_dev(e, slot, e->d_vol.p, S, H, W, flags, e->d_out.p));
    if (out) CU(cudaMemcpyAsync(out, e->d_out.p, n, cudaMemcpyDeviceToHost, e->st));
    CU(cudaEventRecord(e->ev[6], e->st));
    return 0;
  }));
  collect_timings(e);
  return shard_check(e);
}

int lm_fuse(lm_engine* e, const uint8_t* res_l, const uint8_t* res_r, int S, int H, int W, uint8_t* fused, int* spare_value) {
  if (!e || !res_l || !res_r || !fused || !spare_value) return fail(-1, "lm_fuse: NULL argument");
  if (S < 1 || H < 1 || W < 1) return fail(-1, "lm_fuse: empty volume");
  CU(cudaSetDevice(e->device));
  const size_t n = (size_t)S * H * W;
  RC(e->d_out.reserve(n));
  RC(e->d_out2.reserve(n));
  CU(cudaMemcpyAsync(e->d_out.p, res_l, n, cudaMemcpyHostToDevice, e->st));
  CU(cudaMemcpyAsync(e->d_out2.p, res_r, n, cudaMemcpyHostToDevice, e->st));
  RC(fuse_device(e->d_out.p, e->d_out2.p, n, e->d_scratch.p, e->d_spare, e->num_sms, e->st));
  CU(cudaMemcpyAsync(fused, e->d_out.p, n, cudaMemcpyDeviceToHost, e->st));
  int32_t spare = 0;
  CU(cudaMemcpyAsync(&spare, e->d_spare, sizeof(int32_t), cudaMemcpyDeviceToHost, e->st));
  CU(cudaStreamSynchronize(e->st));
  *spare_value = (int)spare;
  return 0;
}

int lm_preprocess(lm_engine* e, const int16_t* vol, int S, int H, int W, int out_h, int out_w, int clip,
                  int16_t* resized, int32_t* boxes) {
  if (!e || !vol || !resized || !boxes) return fail(-1, "lm_preprocess: NULL argument");
  if (S < 1 || H < 1 || W < 1 || out_h < 1 || out_w < 1) return fail(-1, "lm_preprocess: empty volume");
  CU(cudaSetDevice(e->device));
  const size_t n = (size_t)S * H * W, nr = (size_t)S * out_h * out_w;
  RC(e->d_vol.reserve(n));
  RC(e->d_boxes.reserve((size_t)S * 4));
  RC(e->d_resized.reserve(nr));
  CU(cudaMemcpyAsync(e->d_vol.p, vol, n * sizeof(int16_t), cudaMemcpyHostToDevice, e->st));
  RC(launch_bodymask(e->d_vol.p, S, H, W, e->d_boxes.p, nullptr, e->num_sms, e->st));
  RC(launch_resize(e->d_vol.p, S, H, W, e->d_boxes.p, e->d_resized.p, out_h, out_w, clip, e->num_sms, e->st));
  CU(cudaMemcpyAsync(resized, e->d_resized.p, nr * sizeof(int16_t), cudaMemcpyDeviceToHost, e->st));
  CU(cudaMemcpyAsync(boxes, e->d_boxes.p, (size_t)S * 4 * sizeof(int32_t), cudaMemcpyDeviceToHost, e->st));
  CU(cudaStreamSynchronize(e->st));
  return 0;
}

int lm_simple_bodymask(lm_engine* e, const int16_t* slice, int H, int W, uint8_t* mask) {
  if (!e || !slice || !mask) return fail(-1, "lm_simple_bodymask: NULL argument");
  if (H < 1 || W < 1) return fail(-1, "lm_simple_bodymask: empty slice");
  CU(cudaSetDevice(e->device));
  const size_t n = (size_t)H * W;
  RC(e->d_vol.reserve(n));
  RC(e->d_boxes.reserve(4));
  RC(e->d_mask.reserve(n));
  CU(cudaMemcpyAsync(e->d_vol.p, slice, n * sizeof(int16_t), cudaMemcpyHostToDevice, e->st));
  RC(launch_bodymask(e->d_vol.p, 1, H, W, e->d_boxes.p, e->d_mask.p, e->num_sms, e->st));
  CU(cudaMemcpyAsync(mask, e->d_mask.p, n, cudaMemcpyDeviceToHost, e->st));
  CU(cudaStreamSynchronize(e->st));
  return 0;
}

int lm_forward(lm_engine* e, int slot, const int16_t* resized, int S, uint8_t* labels, float* scores) {
  if (!e || !resized || !labels) return fail(-1, "lm_forward: NULL argument");
  if (S < 1) return fail(-1, "lm_forward: S < 1");
  CU(cudaSetDevice(e->device));
  const size_t nr = (size_t)S * R * R;
  RC(e->d_resized.reserve(nr));
  RC(e->d_labels.reserve(nr));
  return run_checked(e, [&]() -> int {
    CU(cudaMemcpyAsync(e->d_resized.p, resized, nr * sizeof(int16_t), cudaMemcpyHostToDevice, e->st));
    RC(forward_all(e, slot, e->d_resized.p, S, e->d_labels.p, scores, nullptr));
    CU(cudaMemcpyAsync(labels, e->d_labels.p, nr, cudaMemcpyDeviceToHost, e->st));
    return 0;
  });
}

int lm_forward_dev(lm_engine* e, int slot, const int16_t* d_resized, int S, uint8_t* d_labels, float* conv_ms) {
  if (!e || !d_resized || !d_labels) return fail(-1, "lm_forward_dev: NULL argument");
  CU(cudaSetDevice(e->device));
  return run_checked(e, [&]() -> int {
    e->launches = 0;
    e->ev_used = 0;
    return forward_all(e, slot, d_resized, S, d_labels, nullptr, conv_ms);
  });
}

int lm_postprocess(lm_engine* e, const uint8_t* labels, int S, int H, int W, const int32_t* spare, int n_spare,
                   int skip_below, uint8_t* out) {
  if (!e || !labels || !out) return fail(-1, "lm_postprocess: NULL argument");
  if (S < 1 || H < 1 || W < 1) return fail(-1, "lm_postprocess: empty volume");
  CU(cudaSetDevice(e->device));
  const size_t n = (size_t)S * H * W;
  RC(e->d_out.reserve(n));
  RC(e->d_out2.reserve(n));
  if (n_spare < 0 || n_spare > 16 || (n_spare > 0 && !spare)) return fail(-1, "lm_postprocess: n_spare %d not in [0,16]", n_spare);
  return run_checked(e, [&]() -> int {
    CU(cudaMemcpyAsync(e->d_out.p, labels, n, cudaMemcpyHostToDevice, e->st));
    int64_t launches = 0;
    // arbitrary label values: the post-processing synchronises once to learn which occur (max_label = -1)
    RC(postprocess_device(e->post, e->d_out.p, S, H, W, spare, n_spare, nullptr, 0, skip_below, -1, e->d_out2.p, e->num_sms, e->st,
                          &launches));
    CU(cudaMemcpyAsync(out, e->d_out2.p, n, cudaMemcpyDeviceToHost, e->st));
    return 0;
  });
}

int lm_keep_largest_component(lm_engine* e, const uint8_t* mask, int S, int H, int W, uint8_t* out) {
  if (!e || !mask || !out) return fail(-1, "lm_keep_largest_component: NULL argument");
  if (S < 1 || H < 1 || W < 1) return fail(-1, "lm_keep_largest_component: empty mask");
  CU(cudaSetDevice(e->device));
  const size_t n = (size_t)S * H * W;
  RC(e->d_out.reserve(n));
  RC(e->d_out2.reserve(n));
  CU(cudaMemcpyAsync(e->d_out.p, mask, n, cudaMemcpyHostToDevice, e->st));
  const int r = keep_largest_component_device(e->post, e->d_out.p, S, H, W, e->d_out2.p, e->num_sms, e->st);
  if (r == -21) return fail(-21, "lm_keep_largest_component: the mask has no foreground (the reference raises IndexError here)");
  RC(r);
  CU(cudaMemcpyAsync(out, e->d_out2.p, n, cudaMemcpyDeviceToHost, e->st));
  CU(cudaStreamSynchronize(e->st));
  return 0;
}

int lm_reshape_masks(lm_engine* e, const uint8_t* masks, int mask_h, int mask_w, const int32_t* boxes, int S, int H,
                     int W, uint8_t* out) {
  if (!e || !masks || !boxes || !out) return fail(-1, "lm_reshape_masks: NULL argument");
  if (S < 1 || H < 1 || W < 1 || mask_h < 1 || mask_w < 1) return fail(-1, "lm_reshape_masks: empty input");
  CU(cudaSetDevice(e->device));
  const size_t n = (size_t)S * H * W, nr = (size_t)S * mask_h * mask_w;
  RC(e->d_labels.reserve(nr));
  RC(e->d_boxes.reserve((size_t)S * 4));
  RC(e->d_out.reserve(n));
  CU(cudaMemcpyAsync(e->d_labels.p, masks, nr, cudaMemcpyHostToDevice, e->st));
  CU(cudaMemcpyAsync(e->d_boxes.p, boxes, (size_t)S * 4 * sizeof(int32_t), cudaMemcpyHostToDevice, e->st));
  RC(reshape_device(e->d_labels.p, e->d_boxes.p, S, H, W, mask_h, mask_w, e->d_out.p, e->num_sms, e->st));
  CU(cudaMemcpyAsync(out, e->d_out.p, n, cudaMemcpyDeviceToHost, e->st));
  CU(cudaStreamSynchronize(e->st));
  return 0;
}

int lm_debug_activation_info(int act_id, int* level, int* channels, int* split) {
  if (act_id < 0 || act_id >= NUM_ACT) return fail(-1, "activation id %d out of range", act_id);
  if (level) *level = ACT[act_id].level;
  if (channels) *channels = ACT[act_id].C;
  if (split) *split = ACT[act_id].split;
  return 0;
}

int lm_debug_read_activation(lm_engine* e, int act_id, int n, float* out) {
  if (!e || !out) return fail(-1, "lm_debug_read_activation: NULL argument");
  if (act_id < 0 || act_id >= NUM_ACT) return fail(-1, "activation id %d out of range", act_id);
  if (n < 1 || n > e->B) return fail(-1, "n out of range");
  CU(cudaSetDevice(e->device));
  const int hw = R >> ACT[act_id].level;
  const size_t per = (size_t)hw * hw * ACT[act_id].C;
  CU(cudaStreamSynchronize(e->st));
  if (!ACT[act_id].split) {
    CU(cudaMemcpy(out, e->act[act_id], (size_t)n * per * sizeof(float), cudaMemcpyDeviceToHost));
    return 0;
  }
  std::vector<op_t> tmp((size_t)n * 2 * per);
  CU(cudaMemcpy(tmp.data(), e->act[act_id], tmp.size() * sizeof(op_t), cudaMemcpyDeviceToHost));
  const float unscale = (e->range_slot >= 0 && e->range_slot < LM_MAX_SLOTS) ? 1.f / e->slots[e->range_slot].act_scale[act_id] : 1.f;
  for (int i = 0; i < n; ++i)
    for (size_t k = 0; k < per; ++k)
      out[(size_t)i * per + k] = ((float)tmp[((size_t)i * 2) * per + k] + (float)tmp[((size_t)i * 2 + 1) * per + k] * kLoUnscale) * unscale;
  return 0;
}

int lm_debug_activation_scale(lm_engine* e, int slot, int act_id, float* scale) {
  if (!e || !scale) return fail(-1, "lm_debug_activation_scale: NULL argument");
  if (slot < 0 || slot >= LM_MAX_SLOTS) return fail(-1, "lm_debug_activation_scale: slot %d out of range", slot);
  if (act_id < 0 || act_id >= NUM_ACT) return fail(-1, "activation id %d out of range", act_id);
  *scale = ACT[act_id].split ? e->slots[slot].act_scale[act_id] : 1.f;
  return 0;
}

int lm_set_option(lm_engine* e, const char* key, int value) {
  if (!e || !key) return fail(-1, "lm_set_option: NULL argument");
  e->graph_epoch++;   // captured forwards bake the kernel choices in
  if (!strcmp(key, "graphs")) { e->use_graphs = value != 0; return 0; }
  if (!strcmp(key, "bn64_mask")) { e->bn64_mask = (unsigned)value; return 0; }   // takes effect at the next lm_load_weights
  if (!strcmp(key, "time_convs")) { e->time_convs = value != 0; e->ev_used = 0; return 0; }
  if (!strcmp(key, "post_debug_stage")) { e->post.debug_stage = value; return 0; }
  if (!strcmp(key, "chunk_kb")) { if (value < 1) return fail(-1, "chunk_kb must be >= 1"); e->chunk_kb = e->chunk_kb_wide = value; return 0; }
  if (!strcmp(key, "weight_mcast")) { if (value != 0 && value != 2) return fail(-1, "weight_mcast must be 0 or 2"); e->weight_mcast = value; return 0; }
  if (!strcmp(key, "conv64_cm")) { if (value != 0 && value != 1) return fail(-1, "conv64_cm must be 0 or 1"); e->conv64_cm = value; return 0; }
  if (!strcmp(key, "stem_v2")) { if (value < 0 || value > 3) return fail(-1, "stem_v2 must be 0, 1, 2 or 3"); e->stem_v2 = value; return 0; }
  if (!strcmp(key, "upsample_v2")) { e->upsample_v2 = value < 0 ? 0 : (value > 2 ? 2 : value); return 0; }
  if (!strcmp(key, "ccl_rule")) { e->post.ccl_rule = value != 0; return 0; }
  if (!strcmp(key, "shard_slab_ccl")) { e->shard_slab_ccl = value != 0; return 0; }
  if (!strcmp(key, "shard_test_slabs")) { if (value < 0 || value > kShardMaxWorld) return fail(-1, "shard_test_slabs out of range"); e->shard_test_slabs = value; return 0; }
  if (!strcmp(key, "merge_ctas")) { if (value < 0) return fail(-1, "merge_ctas must be >= 0"); e->post.merge_ctas = value; return 0; }
  if (!strcmp(key, "post_region_capacity")) {  // test hook: shrink / grow the region tables (exercises the overflow re-run)
    if (value < 1) return fail(-1, "post_region_capacity must be >= 1");
    CU(cudaSetDevice(e->device));
    CU(cudaStreamSynchronize(e->st));
    e->post.release_regions();
    if (e->post.cap_vox) RC(e->post.reserve_regions((uint32_t)value));
    return 0;
  }
  if (!strcmp(key, "chunk_kb_wide")) { if (value < 1) return fail(-1, "chunk_kb_wide must be >= 1"); e->chunk_kb_wide = value; return 0; }
  return fail(-1, "lm_set_option: unknown key %s", key);
}

int lm_last_conv_timing(const lm_engine* e, float* conv_ms, int64_t* conv_launches) {
  if (!e) return fail(-1, "lm_last_conv_timing: NULL engine");
  if (conv_ms) *conv_ms = e->last_conv_ms;
  if (conv_launches) *conv_launches = e->last_conv_launches;
  return 0;
}

int lm_last_timings(const lm_engine* e, float* ms7, int64_t* kernel_launches) {
  if (!e) return fail(-1, "lm_last_timings: NULL engine");
  if (ms7) memcpy(ms7, e->last_ms, sizeof(e->last_ms));
  if (kernel_launches) *kernel_launches = e->launches;
  return 0;
}

}  // extern "C"
