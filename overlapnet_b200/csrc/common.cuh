// common.cuh -- handle, error plumbing and small device helpers shared by all translation units.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <memory>
#include <string>
#include <vector>
#include <map>

#include "../../include/ovn_b200.h"

struct ovn_handle;

namespace ovn {

// The one owner of a cudaMalloc'ed block (cudaHostAlloc'ed when Pinned) of T; frees it on destruction.
// Converts to T* so that kernels and runtime calls take it as a plain pointer.  ensure() is the only place
// where the block and its capacity change; `buf = {}` hands the block to a temporary that frees it.
template <class T, bool Pinned = false>
class Buffer {
 public:
  Buffer() = default;
  Buffer(Buffer&& o) noexcept { swap(o); }
  Buffer& operator=(Buffer&& o) noexcept {
    Buffer old(std::move(o));
    swap(old);
    return *this;
  }
  ~Buffer() {
    if (!p_) return;
    if (Pinned) cudaFreeHost(p_);
    else cudaFree(p_);
  }
  operator T*() const { return p_; }
  T* get() const { return p_; }
  size_t bytes() const { return cap_; }
  // At least `bytes` bytes; a grow frees the old block (cudaFree synchronises the device) and allocates
  // max(bytes, reserve).  On failure the buffer is empty and the CUDA error is consumed, so the handle
  // stays usable.
  int ensure(ovn_handle* h, size_t bytes, size_t reserve = 0);

 private:
  void swap(Buffer& o) {
    std::swap(p_, o.p_);
    std::swap(cap_, o.cap_);
  }
  T* p_ = nullptr;
  size_t cap_ = 0;
};
template <class T> using PinnedBuffer = Buffer<T, true>;

// Head of ovn_handle::h_pinned, the pinned staging of the host entry points; the candidate indices, overlaps
// and yaws of ovn_query_cloud_vs_bank_host follow it (ovn_handle::stage_*).
struct StageHeader {
  int32_t err;                   // ovn_handle::d_err, copied back by check_device_error
  int32_t pad0[3];
  int64_t offsets[2];            // point offsets of the one staged cloud
  int64_t pad1[2];
  float loss[3];                 // ovn_head_gradients: total, overlap, orientation
  int32_t pad2;
};
static_assert(offsetof(StageHeader, offsets) == 16 && offsetof(StageHeader, loss) == 48 && sizeof(StageHeader) == 64,
              "pinned staging layout");
static_assert(sizeof(float) == sizeof(int32_t), "the three staging arrays are 4 B per pair");

constexpr int kFeatC = 128;           // leg output channels (generateNet.py:214)
constexpr int kMaxLegLayers = 12;
enum ProfKind { PROF_DELTA = 0, PROF_CONV2, PROF_CONV3, PROF_CORR, PROF_SCATTER, PROF_GATHER, PROF_LEG, PROF_GATHER_ROWS,
                PROF_ROWS_TOPK, PROF_PGO, PROF_RENDER_SCATTER, PROF_RENDER_GATHER, PROF_SURFEL_BUILD, PROF_SURFEL_SCATTER,
                PROF_SURFEL_GATHER, kProfKinds };

// The one owner of another process's shard mapped by ovn_shard_open (cudaIpcOpenMemHandle); unmaps it on
// destruction.  Move-only, like Buffer.
class IpcMapping {
 public:
  IpcMapping() = default;
  explicit IpcMapping(void* p) : p_(p) {}
  IpcMapping(IpcMapping&& o) noexcept { std::swap(p_, o.p_); }
  IpcMapping& operator=(IpcMapping&& o) noexcept {
    IpcMapping old(std::move(o));
    std::swap(p_, old.p_);
    return *this;
  }
  ~IpcMapping() {
    if (p_) cudaIpcCloseMemHandle(p_);
  }
  void* get() const { return p_; }

 private:
  void* p_ = nullptr;
};

struct ConvSpec {                      // one Conv2D layer (valid padding, bias)
  char name[24];
  int kh, kw, sh, sw, cin, cout;
  int relu;
  int h_in, w_in, h_out, w_out;
};

struct LayerWeights {
  std::vector<float> kernel;           // Keras layout, flattened
  std::vector<int64_t> dims;
  std::vector<float> bias;
  bool set = false;
};

}  // namespace ovn

namespace ovn {
struct TcState;
struct TcStateDelete { void operator()(TcState* t) const; };   // network_tc.cu: TcState is private to it

// The flat parameter vector of training (ovn_copy_gradients' layout): c_conv1..3, overlap_output, then the leg
// layers from input to output, each [K + 1][N] floats (the kernel [K][N] in Keras layout, then the bias [N]).
// Set by ovn_create from the layer shapes.
struct ParamLayout {
  int64_t off[kMaxLegLayers + 4] = {};        // by weight slot (the index of d_w / d_b): the layer's kernel
  int64_t n_kernel[kMaxLegLayers + 4] = {};   // K N: the layer's bias starts at off + n_kernel
  int64_t n_head = 0;                         // the heads' prefix
  int64_t n_total = 0;                        // the whole network
};
// weight slot of the i-th layer of the flat vector
inline int flat_slot(int i) { return i < 4 ? kMaxLegLayers + i : i - 4; }

// Which layers the last valid gradients (TrainState::grad) cover
enum GradCover { kNoGrads = 0, kHeadGrads, kNetGrads };

// Training (fp32 handles; allocated when a handle first trains, sized by max_batch_pairs).  The gradients and
// Adagrad accumulators are whole ParamLayout vectors: a head-only call leaves the leg's part of grad unused.
struct TrainState {
  Buffer<float> x4;             // [max_batch_pairs][dense_in] c_conv3 output, then dL/d(its pre-activation)
  Buffer<float> dx3;            // [max_batch_pairs][24][24][128] dL/dx3, then dL/d(pre-activation of c_conv2)
  Buffer<float> corr;           // [max_batch_pairs][Wf] orientation logits
  Buffer<float> overlap;        // [max_batch_pairs]
  Buffer<float> dz;             // [max_batch_pairs] dL/d(Dense logit)
  Buffer<int32_t> yaw;          // [max_batch_pairs]
  Buffer<float> w3t;            // c_conv3 kernel with in / out swapped
  Buffer<float> part;           // split-K partials of the weight gradients
  Buffer<float> grad;           // [ParamLayout::n_total]
  Buffer<float> accum;          // [ParamLayout::n_total] Adagrad accumulators
  Buffer<float> loss;           // [3] total, overlap, orientation
  Buffer<float> chunk_loss;     // [64][3] the losses of each chunk of a *_gradients_chunks call
  PinnedBuffer<float> chunk_loss_host;
  GradCover grads = kNoGrads;   // set by the last successful ovn_head_gradients / ovn_net_gradients
  // Whole-network training (ovn_net_gradients): allocated on its first call, grown to the batch.  The 2n images
  // of an n-pair batch are LEFT 0..n-1, then RIGHT 0..n-1.
  Buffer<float> images;         // [2n][H][W][C] the gathered input images
  Buffer<float> acts;           // every leg layer's output for those images, layer after layer
  Buffer<float> dact[2];        // ping-pong gradients of the leg activations (dact[0] first holds dL/d(volumes))
  Buffer<float> dfv_part;       // k_delta_dgrad partials: LEFT [n][nb][Wf][128], then RIGHT [n][row tiles][Wf][128]
  Buffer<float> dcorr;          // [n][Wf] dL/d(correlation logits)
  Buffer<int32_t> pair_rows;    // [2n] 0..2n-1: LEFT / RIGHT rows of the batch's volumes
  Buffer<float> wt;             // a leg kernel with in / out swapped
  int64_t net_fv_off = 0;       // the last ovn_net_gradients batch: its volumes [2 net_np][Wf][128] at acts + net_fv_off
  int net_np = 0;
  // Stage readback (ovn_set_train_stop / ovn_copy_train_stage).  stop_*: the point where the next gradient call
  // stops, -1 = none; consumed by that call.  stopped: the running call reached it.  The stages of the last
  // gradient call: its pairs (0 = none), its flow and where it stopped (-1 = it ran to the end).
  int stop_stage = -1, stop_layer = -1;
  bool stopped = false;
  const float* stop_buf = nullptr;   // the live buffer of the stage the call stopped at
  int stage_np = 0;
  bool stage_net = false;
  int stage_stop = -1, stage_stop_layer = -1;
};
// true when the running gradient call stops at (stage, layer), whose value is in `live`, or has stopped before
inline bool train_stop_here(TrainState& t, int stage, int layer, const float* live) {
  if (!t.stopped && t.stop_stage == stage && t.stop_layer == layer) {
    t.stopped = true;
    t.stop_buf = live;
  }
  return t.stopped;
}

// Monte Carlo localization (ovn_mcl_*, mcl.cu).  The map: K keyframes' planar poses and the raster of the nearest
// keyframe per cell; the particles: two structure-of-arrays float64 buffers of 4 cap values (x, y, theta, log-weight).
struct McMap {
  int K = 0, rows = 0, cols = 0;
  double x0 = 0.0, y0 = 0.0, cell = 0.0;
};
struct McParticles {
  double *x, *y, *th, *lw;
};
// the device scalars of one update: k_mcl_final writes them, the host reads [0, kScTouched); OVN_MCL_STAGE_SCALARS
// copies [kScMax, kScU0]
enum McScalar { kScMax = 0, kScExpSum, kScEss, kScX, kScY, kScTheta, kScResample, kScU0, kScRefused, kScTouched,
                kScCount };
constexpr int kMcPartialStride = 8;      // doubles per block partial
constexpr int kMcMaxParticles = 1 << 24;
constexpr int kMcMaxKeyframes = 1 << 24;
constexpr int64_t kMcMaxCells = int64_t(1) << 28;
enum McHeld { kMcHeldPredict = 1, kMcHeldUpdate = 2, kMcHeldResample = 4 };   // the stages McState holds
struct McState {
  McMap map;
  Buffer<double> kf;             // [K][3] x, y, theta of the keyframes
  Buffer<int32_t> raster;        // [rows][cols] keyframe index or -1
  Buffer<int32_t> flags;         // [K] touched by the last predict
  Buffer<int32_t> slot;          // [K] position in the last predict's touched list, or -1
  Buffer<double> part[2];        // particle buffers, [4][cap]
  Buffer<int32_t> kidx;          // [cap] the last lookup
  Buffer<double> ll, w, cdf;     // [cap] log-likelihood, normalised weights, inclusive prefix sum of the weights
  Buffer<int32_t> anc;           // [cap] the last resampling's ancestors
  Buffer<double> tiles;          // prefix sum: one total per tile
  Buffer<double> partial;        // [kMclRedBlocks][kMcPartialStride] per-block partials of a reduction
  Buffer<double> scal;           // [kScCount] McScalar
  PinnedBuffer<double> host;     // [kScCount] their host copy
  int cap = 0;                   // particles the buffers hold
  int n = 0;                     // particles of the set, 0 before ovn_mcl_init
  int cur = 0, pred_buf = 0;     // the buffer of the current set; the one the last predict moved
  uint64_t seed = 0;
  int64_t step = 0;              // predicts since ovn_mcl_init
  int pending = -1;              // n_touched of a predict that awaits its update, else -1
  int stages = 0;                // McHeld bits
};
}  // namespace ovn

struct ovn_handle {
  ovn_config cfg;
  int device = 0;
  int sm_count = 0;
  std::string last_error;
  int64_t launches = 0;

  int C = 0;                            // input channels (infer.py:61-73)
  int n_leg = 0;
  ovn::ConvSpec leg[ovn::kMaxLegLayers];
  ovn::ConvSpec head[3];                // c_conv1..3 in "delta image" coordinates
  int o1_h = 0, o1_w = 0;               // c_conv1 output (360, 24)
  int o2_h = 0, o2_w = 0;               // c_conv2 output (24, 24)
  int o3_h = 0, o3_w = 0;               // c_conv3 output (22, 22)
  int dense_in = 0;
  ovn::ParamLayout params;              // the flat gradient / accumulator layout of training

  std::map<std::string, ovn::LayerWeights> host_w;
  bool weights_ready = false;
  bool net_ok = false;                 // leg/head shapes valid for this config (else projection only)
  std::string net_error;

  // device weights, fp32 GEMM layout [K][N] (K = kh*kw*cin, Keras HWIO flattened is already that)
  ovn::Buffer<float> d_w[ovn::kMaxLegLayers + 4];
  ovn::Buffer<float> d_b[ovn::kMaxLegLayers + 4];

  // workspaces, allocated by ovn_create unless noted
  ovn::Buffer<unsigned long long> d_keys;    // [max_batch_scans][H*W] atomic-min keys; twice that with probability
                                             //   channels (the two key images of ovn_preprocess_cues_batch)
  ovn::Buffer<unsigned long long> d_pair_keys; // ovn_gt_pairs_count: [tile_cur][tile_ref][H*W] keys, grown on use
  ovn::Buffer<uint8_t> d_pair_prune;         // ovn_gt_pairs_count: pruned-pair counter + [n_cur][n_ref] flags, grown on use
  ovn::Buffer<uint32_t> d_valid_words;       // validity bitmask, 1 bit per point; these three grow with the points
  ovn::Buffer<uint32_t> d_word_prefix;       //   of projections that return per-point indices
  ovn::Buffer<uint32_t> d_scan_tmp;          //   (exclusive prefix of popcounts, block sums)
  ovn::Buffer<float> d_act[2];               // fp32 only: ping-pong activations of the leg
  ovn::Buffer<float> d_input;                // [max_batch_scans][H][W][C]
  ovn::Buffer<float> d_o1;                   // fp32 only: [max_batch_pairs][360][24][64]
  ovn::Buffer<float> d_o2;                   // fp32 only: [max_batch_pairs][24][24][128]
  ovn::Buffer<float> d_G;                    // fp32 only: [max_batch_pairs][360][360] correlation Gram matrices
  ovn::Buffer<int32_t> d_cand_idx;           // [max_batch_pairs] candidate indices of ovn_heads_1vsN / the host query
  ovn::Buffer<int32_t> d_idx_san;            // [max_batch_pairs] x3 bounds-checked (clamped) copies of the caller's index lists
  ovn::Buffer<int> d_err;                    // device error flag: 0 or an ovn::DeviceError
  cudaEvent_t ev_bank = nullptr;             // recorded after ovn_bank_prepare: the host entry points (own stream) wait on it
  // ovn_query_cloud_vs_bank_host / ovn_encode_clouds_host
  ovn::Buffer<float> d_query_fv;             // [360][128]
  ovn::Buffer<float> d_query_overlap;        // [max_batch_pairs]
  ovn::Buffer<int32_t> d_query_yaw;          // [max_batch_pairs]
  ovn::Buffer<float> d_stage_points;         // staged clouds, grown on use
  ovn::Buffer<int64_t> d_stage_offsets;      // [max_batch_scans + 1], allocated on first use
  ovn::PinnedBuffer<uint8_t> h_pinned;       // StageHeader, then candidate indices / overlaps / yaws [max_batch_pairs]
  // ovn_rows_topk / ovn_heads_prefix_topk, allocated on first use
  ovn::Buffer<uint8_t> d_topk_rows;          // one k_rows_topk launch's row offsets (int64) then row lengths (int32)
  ovn::Buffer<uint8_t> d_topk_scratch;       // ovn_heads_prefix_topk: kTopkScratchPairs overlaps (f32), then yaws (i32)
  // a sharded training image bank (ovn_shard_*): this process's shards, then the other processes' shards it
  // mapped.  Declared in this order so that the mappings are closed before the own shards are freed.
  std::vector<ovn::Buffer<uint8_t>> own_shards;
  std::vector<ovn::IpcMapping> open_shards;
  ovn::McState mcl;                          // ovn_mcl_*: map and particles, allocated by ovn_mcl_set_map / ovn_mcl_init
  ovn::Buffer<uint8_t> d_pgo;                // ovn_pgo_optimize_host: one call's inputs and workspace, grown on use
  // where the last successful ovn_pgo_optimize_host call put its graphs and its arrays (ovn_pgo_array order) in
  // d_pgo, for ovn_pgo_copy_workspace; pgo_node_off is empty when there is no such call
  std::vector<int64_t> pgo_node_off, pgo_edge_off;
  size_t pgo_array_off[15] = {};
  ovn::Buffer<uint8_t> d_render;             // ovn_render_*: one call's entry table, grown on use
  ovn::Buffer<uint8_t> d_surfel;             // ovn_surfels_batch: one call's projection images, grown on use
  cudaStream_t own_stream = nullptr;
  // per-kernel profiling (ovn_profile_enable / ovn_profile_read)
  bool profiling = false;
  std::vector<cudaEvent_t> prof_ev[ovn::kProfKinds];   // start/stop pairs, in launch order
  std::unique_ptr<ovn::TcState, ovn::TcStateDelete> tc;   // tensor-core path state (network_tc.cu)
  std::unique_ptr<ovn::TrainState> train;  // overlap-head training state (network_fp32.cu), NULL until first used
  int32_t train_precision = OVN_TRAIN_FP32;  // ovn_set_train_precision
  bool train_tc = false;                   // inside ovn_head_gradients / ovn_net_gradients at OVN_TRAIN_TF32X3:
                                           // launch_gemm and the |l - r| backward take their 3xTF32 kernels
  bool dgrad_tc_smem = false;              // k_delta_dgrad_tc's dynamic shared-memory limit is raised on this device

  ~ovn_handle();                           // the streams and events; the buffers free themselves
  ovn::StageHeader* stage() const { return reinterpret_cast<ovn::StageHeader*>(h_pinned.get()); }
  int32_t* stage_cand_idx() const { return reinterpret_cast<int32_t*>(h_pinned + sizeof(ovn::StageHeader)); }
  float* stage_overlap() const { return reinterpret_cast<float*>(stage_cand_idx() + cfg.max_batch_pairs); }
  int32_t* stage_yaw() const { return reinterpret_cast<int32_t*>(stage_overlap() + cfg.max_batch_pairs); }
};

#define OVN_SET_ERR(h, code, ...)                                 \
  do {                                                            \
    char _buf[512];                                               \
    snprintf(_buf, sizeof(_buf), __VA_ARGS__);                    \
    (h)->last_error = _buf;                                       \
    return (code);                                                \
  } while (0)

// A failed runtime call is reported once: its error is consumed, so the next OVN_LAUNCH_CHECK does not blame
// a kernel launch for it.
#define OVN_CUDA(h, call)                                                                   \
  do {                                                                                      \
    cudaError_t _e = (call);                                                                \
    if (_e != cudaSuccess) {                                                                \
      cudaGetLastError();                                                                   \
      OVN_SET_ERR(h, OVN_ERR_CUDA, "%s failed at %s:%d: %s", #call, __FILE__, __LINE__,     \
                  cudaGetErrorString(_e));                                                  \
    }                                                                                       \
  } while (0)

#define OVN_LAUNCH_CHECK(h)                                                                 \
  do {                                                                                      \
    (h)->launches++;                                                                        \
    cudaError_t _e = cudaGetLastError();                                                    \
    if (_e != cudaSuccess) {                                                                \
      OVN_SET_ERR(h, OVN_ERR_CUDA, "kernel launch failed at %s:%d: %s", __FILE__, __LINE__, \
                  cudaGetErrorString(_e));                                                  \
    }                                                                                       \
  } while (0)

namespace ovn {

template <class T, bool Pinned>
int Buffer<T, Pinned>::ensure(ovn_handle* h, size_t bytes, size_t reserve) {
  if (bytes <= cap_) return OVN_OK;
  *this = {};                           // free the old block first: the new one may need its memory
  if (reserve < bytes) reserve = bytes;
  void* p = nullptr;
  if (Pinned) OVN_CUDA(h, cudaHostAlloc(&p, reserve, cudaHostAllocDefault));
  else OVN_CUDA(h, cudaMalloc(&p, reserve));
  p_ = static_cast<T*>(p);
  cap_ = reserve;
  return OVN_OK;
}

// Every ABI entry point runs on the device its handle was created on (ADVICE r1: Engine(device=1)
// with another current device allocated on the wrong GPU).
struct DeviceGuard {
  int prev = -1;
  bool switched = false;
  explicit DeviceGuard(const ovn_handle* h) {
    if (h && cudaGetDevice(&prev) == cudaSuccess && prev != h->device) switched = cudaSetDevice(h->device) == cudaSuccess;
  }
  ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
};

// Every value a kernel writes to ovn_handle::d_err (0: no error); check_device_error maps each to a status and
// a message.  The numbers appear in messages, so they do not change.
enum DeviceError : int {
  // a bounded wait on an mbarrier ring timed out: 1xx in the producer, 2xx / 4xx in a consumer
  kErrDeltaLeftProducer = 101, kErrDeltaLeftConsumer = 402,      // k_delta_conv1_wgmma: LEFT volume
  kErrDeltaRightProducer = 103, kErrDeltaRightConsumer = 404,    //   RIGHT window
  kErrDeltaW1Producer = 102, kErrDeltaW1Consumer = 202,          //   W1 groups
  kErrDeltaO1Producer = 104, kErrDeltaO1Consumer = 405,          //   o1 staging (the store lane / the writers)
  kErrConv2Producer = 111, kErrConv2Consumer = 211,              // k_conv2_wgmma: o1 + W2 stages
  kErrConv3X3Producer = 121, kErrConv3X3Consumer = 221,          // k_conv3_wgmma: x3 rows
  kErrConv3W3Producer = 122, kErrConv3W3Consumer = 222,          //   W3 slabs
  kErrCorrRightProducer = 131, kErrCorrRightConsumer = 231,      // k_corr_wgmma: RIGHT third
  kErrCorrLeftProducer = 132, kErrCorrLeftConsumer = 232,        //   LEFT tiles
  kErrInjectedFault = 501,        // k_conv2_wgmma under OVN_DEBUG_FAULT (the error-path test hook)
  kErrBadIndex = 900,             // a pair / candidate index outside [0, bank_size)
  kErrRowNotPrepared = 901,       // resident bank: the row was never passed to ovn_bank_prepare
  kErrIcpBadIndex = 902,          // ovn_icp_pairs: a scan index outside [0, n_scans)
  kErrNonFiniteOperand = 910,     // an fp16 operand of the tensor-core heads or leg is not finite (NaN, inf, > 65504)
  kErrPeerWait = 950,             // ovn_peer_wait: a peer rank never signalled
};

// RAII-free profiling helpers: record an event on `s` before / after a launch when enabled
inline void prof_mark(ovn_handle* h, int kind, cudaStream_t s) {
  if (!h->profiling) return;
  cudaEvent_t e;
  if (cudaEventCreate(&e) != cudaSuccess) return;
  cudaEventRecord(e, s);
  h->prof_ev[kind].push_back(e);
}

// dst = a device copy of v, in a fresh block: freeing the old one synchronises the device, so no queued
// kernel still reads it while it is overwritten
template <class T>
int upload_vec(ovn_handle* h, Buffer<T>& dst, const std::vector<T>& v) {
  dst = {};
  const int rc = dst.ensure(h, v.size() * sizeof(T));
  if (rc != OVN_OK) return rc;
  OVN_CUDA(h, cudaMemcpy(dst, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  return OVN_OK;
}

// ---- stage entry points implemented in the .cu files (called from api.cu) -------------------
int project_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int n_scans,
                  int64_t n_total, float max_range, float* d_range, float* d_vertex,
                  float* d_intensity, int32_t* d_idx, cudaStream_t s);
int normals_batch(ovn_handle* h, const float* d_range, const float* d_vertex, int n_scans,
                  float* d_normal, cudaStream_t s);
int semantic_batch(ovn_handle* h, const int32_t* d_idx, const float* d_probs,
                   const int64_t* d_offsets, int n_scans, int n_classes, float* d_out,
                   cudaStream_t s);
int preprocess_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int n_scans,
                     int64_t n_total, const float* d_probs, float* d_input, cudaStream_t s);
int preprocess_cues_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int n_scans,
                          int64_t n_total, const float* d_probs, float* d_input, cudaStream_t s);
int gt_range_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int n_scans, int64_t n_total,
                   const double* d_pose_ref, const double* d_pose_cur_inv, float max_range, float* d_range,
                   cudaStream_t s);
int gt_overlap_count(ovn_handle* h, const float* d_ref, const float* d_cur, int n_scans, int32_t* d_counts, cudaStream_t s);
int gt_scan_radius(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int n_scans, double* d_radius,
                   cudaStream_t s);
int gt_pairs_count(ovn_handle* h, const float* d_points, const int64_t* h_offsets, int n_ref, const double* d_pose_ref,
                   const double* d_radius, const float* d_cur_range, const double* d_pose_cur_inv, int n_cur,
                   float max_range, int tile_cur, int tile_ref, int32_t* d_counts, int64_t ld_counts,
                   int64_t* d_n_pruned, cudaStream_t s);
// the render (projection.cu): checks the host tables itself, before anything is launched
int render_batch(ovn_handle* h, const float* d_points, const int64_t* h_offsets, int n_clouds, int n_virtual,
                 const int64_t* h_entry_offsets, const int32_t* h_entry_cloud, const double* h_entry_pose,
                 float max_range, float* d_range, float* d_vertex, float* d_intensity, int32_t* d_winner,
                 cudaStream_t s);
int render_preprocess_batch(ovn_handle* h, const float* d_points, const int64_t* h_offsets, int n_clouds,
                            int n_virtual, const int64_t* h_entry_offsets, const int32_t* h_entry_cloud,
                            const double* h_entry_pose, float* d_input, cudaStream_t s);
// surfels and their renders (projection.cu); the parameters are checked by the entry points
int surfels_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int n_scans, int64_t n_total,
                  const ovn_surfel_params& prm, float* d_surfels, cudaStream_t s);
int render_surfels_batch(ovn_handle* h, const float* d_surfels, int n_clouds, const double* d_rays, int n_virtual,
                         const int64_t* h_entry_offsets, const int32_t* h_entry_cloud, const double* h_entry_pose,
                         const ovn_surfel_params& prm, float max_range, float* d_range, float* d_vertex,
                         float* d_intensity, int32_t* d_winner, cudaStream_t s);
int render_surfels_preprocess_batch(ovn_handle* h, const float* d_surfels, int n_clouds, const double* d_rays,
                                    int n_virtual, const int64_t* h_entry_offsets, const int32_t* h_entry_cloud,
                                    const double* h_entry_pose, const ovn_surfel_params& prm, float* d_input,
                                    cudaStream_t s);
int pack_input(ovn_handle* h, const float* d_depth, const float* d_normal, const float* d_prob,
               const float* d_intensity, int n_scans, float* d_input, cudaStream_t s);

int leg_forward_fp32(ovn_handle* h, const float* d_input, int n, float* d_fv, cudaStream_t s);
// the heads_forward_* score n <= max_batch_pairs pairs (heads_dispatch cuts larger calls into such chunks)
int heads_forward_fp32(ovn_handle* h, const float* d_bank, const float* d_query,
                       const int32_t* d_left, const int32_t* d_right, int n, float* d_overlap,
                       int32_t* d_yaw, float* d_corr, cudaStream_t s);

// The most parts of one ovn_adagrad_step_sum, and the most chunks of one *_gradients_chunks call
constexpr int kMaxSumParts = 64;

// Where a gradient call leaves its results.  Chunk c is the pairs [off[c], off[c + 1]) of the call: its flat
// gradients go to grad + c * stride and its losses to loss[3 c .. 3 c + 2] (device), exactly as a call on those
// pairs alone would compute them.  ovn_head_gradients / ovn_net_gradients are one chunk: off = {0, np},
// grad = TrainState::grad, loss = TrainState::loss.  An empty chunk is skipped (the caller zeroes its results).
struct GradChunks {
  int n = 1;
  int off[kMaxSumParts + 1] = {};
  float* grad = nullptr;
  int64_t stride = 0;
  float* loss = nullptr;
  __host__ __device__ int size(int c) const { return off[c + 1] - off[c]; }
};

// training of the overlap head (network_fp32.cu)
int train_alloc(ovn_handle* h);
int head_gradients_fp32(ovn_handle* h, const float* d_bank, const int32_t* left, const int32_t* right, int np,
                        const float* d_gt_overlap, const int32_t* d_gt_orientation, float min_overlap,
                        const GradChunks& ch, cudaStream_t s);
// training of the whole network (network_fp32.cu): left / right index the image bank and are bounds-checked
int net_gradients_fp32(ovn_handle* h, const float* d_images, const int32_t* left, const int32_t* right, int np,
                       const float* d_gt_overlap, const int32_t* d_gt_orientation, float min_overlap,
                       float* d_fv_grad, const GradChunks& ch, cudaStream_t s);
int net_max_pairs(const ovn_handle* h);   // largest n_pairs of one ovn_net_gradients call (launch grid limits)
int64_t train_workspace_bytes(const ovn_handle* h, bool whole_network, int np);   // ovn_train_workspace_bytes
int copy_net_volumes_fp32(ovn_handle* h, float* d_out, cudaStream_t s);
// ovn_train_stage_size / ovn_copy_train_stage: the floats of a stage of the last gradient call, and a copy of them
// (the caller has checked that the stage is held)
int64_t train_stage_floats(const ovn_handle* h, int stage, int layer);
int copy_train_stage_fp32(ovn_handle* h, int stage, int layer, float* d_out, cudaStream_t s);
// The Adagrad step of the heads' (or with whole_network every layer's) prefix of the flat vector, from the
// weighted sum of d_parts [n_parts][that length]: one launch
int adagrad_sum_fp32(ovn_handle* h, bool whole_network, const float* d_parts, int n_parts, const float* h_weights,
                     float lr, cudaStream_t s);
// yaw augmentation of training images (projection.cu): rows are bounds-checked on the device (kErrBadIndex)
int gather_images(ovn_handle* h, const float* d_images, int64_t n_images, const int32_t* d_rows,
                  const int32_t* d_shift, const float* d_rot, int n, float* d_out, cudaStream_t s);
// rows of a sharded image bank (bank_shard.cu): d_dst + i row_bytes = row_bytes bytes at h_src[i], one launch of
// k_gather_rows per kGatherRowsCap rows; the caller has checked every pointer and row_bytes % 16 == 0
constexpr int kGatherRowsCap = 1024;
int gather_rows(ovn_handle* h, const void* const* h_src, int n, int64_t row_bytes, void* d_dst, cudaStream_t s);

// the best k <= kTopkMax records of each row (rows_topk.cu): row r is the h_len[r] overlaps / yaws at h_off[r]
// (element offsets into d_ov / d_yaw, host arrays); one k_rows_topk launch per kTopkRowsPerLaunch rows.  The
// caller has checked k and every length.
constexpr int kTopkMax = 32;
constexpr int64_t kTopkRowsPerLaunch = 65536;
constexpr int64_t kTopkScratchPairs = int64_t(1) << 21;   // ovn_heads_prefix_topk's scratch: 16 MiB
int rows_topk(ovn_handle* h, const float* d_ov, const int32_t* d_yaw, const int64_t* h_off, const int32_t* h_len,
              int64_t rows, int k, float* d_top_ov, int32_t* d_top_idx, int32_t* d_top_yaw, cudaStream_t s);

// Monte Carlo localization (mcl.cu); the caller has checked every argument and the handle's state
int mcl_init(ovn_handle* h, int mode, int n, uint64_t seed, const double* pose, const double* sigma, double radius,
             cudaStream_t s);
int mcl_predict(ovn_handle* h, const double* odom, const double* sigma, int32_t* d_touched, int32_t* n_touched,
                cudaStream_t s);
int mcl_update(ovn_handle* h, const float* d_ov, const int32_t* d_yaw, double s_o, double s_psi, double rho,
               ovn_mcl_estimate* est, cudaStream_t s);
int mcl_copy_particles(ovn_handle* h, double* d_out, cudaStream_t s);
int mcl_copy_stage(ovn_handle* h, int stage, void* d_out, cudaStream_t s);
int mcl_philox(ovn_handle* h, uint64_t seed, const uint32_t* d_ctr, int n, uint32_t* d_out, cudaStream_t s);

// point-to-plane ICP of np pairs (icp.cu), one k_icp_pairs launch; the caller has checked every argument
int icp_pairs(ovn_handle* h, const float* d_vertex, const float* d_normal, int n_scans, const int32_t* d_src,
              const int32_t* d_dst, const double* d_init, int np, const ovn_icp_params& prm, ovn_icp_result* d_out,
              int32_t* d_assoc, double* d_system, cudaStream_t s);

// pose-graph optimization of n_graphs graphs (pose_graph.cu), one k_pgo_graphs launch between the host copies; the
// caller has checked every argument
int pgo_graphs(ovn_handle* h, int n_graphs, const int64_t* node_off, const int64_t* edge_off, const double* poses,
               const int32_t* edge_nodes, const double* edge_pose, const double* edge_weight,
               const ovn_pgo_params& prm, double* out_poses, ovn_pgo_result* out_result, double* out_chi2,
               double* out_scale, double* out_gradient, ovn_pgo_trial* out_trace, cudaStream_t s);
// h_out = array `array` of graph `graph` of the call pgo_graphs recorded; the caller has checked both
int pgo_copy_workspace(ovn_handle* h, int array, int graph, double* h_out);

int corr_forward_fp32(ovn_handle* h, const float* d_bank, const float* d_query, const int32_t* left,
                      const int32_t* right, int np, int32_t* d_yaw, float* d_corr, cudaStream_t s);

// leg layers 0 .. stop_layer of n <= max_batch_scans scans; the last layer writes d_fv, the others hi / lo planes
int leg_forward_tc(ovn_handle* h, const float* d_input, int n, float* d_fv, cudaStream_t s, int stop_layer = kMaxLegLayers);
int tc_leg_stage(ovn_handle* h, const float* d_input, int n, int layer, float* d_hi, float* d_lo, cudaStream_t s);
int heads_forward_tc(ovn_handle* h, const float* d_bank, const float* d_query,
                     const int32_t* d_left, const int32_t* d_right, int n, float* d_overlap,
                     int32_t* d_yaw, float* d_corr, cudaStream_t s);
int tc_pack_weights(ovn_handle* h);
int tc_bank_prepare(ovn_handle* h, const float* d_bank, int64_t capacity, int64_t first, int64_t count, cudaStream_t s);
int tc_bank_release(ovn_handle* h, const float* d_bank);
int tc_set_center(ovn_handle* h, const float* h_mu);
int tc_get_center(ovn_handle* h, float* h_mu, int32_t* is_set);
int tc_calibrate(ovn_handle* h, const float* d_volume, cudaStream_t s);
int tc_copy_heads_stage(ovn_handle* h, int stage, int64_t first, int64_t count, float* d_out, cudaStream_t s);
int64_t tc_heads_stage_pairs(const ovn_handle* h);   // pairs whose stages ovn_copy_heads_stage can copy
// bounds-checked copies of index lists (d_idx_san): out-of-range entries are clamped and flagged in d_err; with
// row_bad (a resident bank's marks), an index whose row is marked raises kErrNonFiniteOperand
int sanitize_indices(ovn_handle* h, const int32_t* d_in, int n, int64_t limit, int code, int32_t* d_out, cudaStream_t s,
                     const int32_t* row_bad = nullptr);
// read (and clear) the device error flag after the caller has synchronised `s`; maps it to a status
int check_device_error(ovn_handle* h, cudaStream_t s);

}  // namespace ovn
