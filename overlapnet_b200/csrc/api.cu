// api.cu -- the C ABI declared in include/ovn_b200.h: handle lifetime, weights, stage dispatch
// and the host-buffer convenience entry points.  No CPU fallback exists anywhere in this library:
// without an sm_90 (Hopper) device ovn_create fails with OVN_ERR_NO_DEVICE.
#include "common.cuh"
#include <math.h>
#include <string.h>
#include <algorithm>

using namespace ovn;

static const char* kLegNames[] = {"s_conv1", "s_conv2", "s_conv3", "s_conv3a", "s_conv4", "s_conv5",
                                  "s_conv6", "s_conv7", "s_conv8", "s_conv9", "s_conv10"};

static void set_spec(ConvSpec& L, const char* name, int kh, int kw, int sh, int sw, int cin, int cout, int relu,
                     int h_in, int w_in) {
  memset(&L, 0, sizeof(L));
  snprintf(L.name, sizeof(L.name), "%s", name);
  L.kh = kh; L.kw = kw; L.sh = sh; L.sw = sw; L.cin = cin; L.cout = cout; L.relu = relu;
  L.h_in = h_in; L.w_in = w_in;
  L.h_out = (h_in - kh) / sh + 1;
  L.w_out = (w_in - kw) / sw + 1;
}

// kernel and bias sizes of the layer in weight slot `slot`
static void slot_sizes(const ovn_handle* h, int slot, int64_t* n_kernel, int64_t* n_bias) {
  if (slot == kMaxLegLayers + 3) {   // overlap_output
    *n_kernel = h->dense_in; *n_bias = 1;
    return;
  }
  const ConvSpec& L = slot < kMaxLegLayers ? h->leg[slot] : h->head[slot - kMaxLegLayers];
  *n_kernel = (int64_t)L.kh * L.kw * L.cin * L.cout;
  *n_bias = L.cout;
}

static __global__ void k_iota(int32_t* p, int n, int start) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = start + i;
}

static __global__ void k_sanitize_idx(const int32_t* __restrict__ in, int32_t* __restrict__ out, int n, int64_t limit,
                                      int code, const int32_t* __restrict__ row_bad, int* __restrict__ err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t v = in[i];
  if (v < 0 || v >= limit) {
    atomicCAS(err, 0, code);              // the first error wins; results of this call are poisoned by the finalize kernels
    v = v < 0 ? 0 : limit - 1;
  }
  if (row_bad && row_bad[v]) atomicCAS(err, 0, kErrNonFiniteOperand);
  out[i] = (int32_t)v;
}

// ---- device-side signalling between the ranks of a sharded bank (search.py transport 'symm') ----------
// Flags are int32 slots in symmetric (peer-mapped) memory holding the number of the last finished step.
// One launch signals every peer (release at system scope, after everything this stream did before),
// one launch waits for every peer (acquire at system scope, bounded).
struct PeerPtrs { int32_t* p[16]; };

static __global__ void k_peer_signal(PeerPtrs dst, int n, int value) {
  const int i = threadIdx.x;
  if (i >= n || dst.p[i] == nullptr) return;
  __threadfence_system();
  asm volatile("st.release.sys.global.s32 [%0], %1;" :: "l"(dst.p[i]), "r"(value) : "memory");
}

static __global__ void k_peer_wait(const int32_t* __restrict__ flags, int n, int skip, int value, int* __restrict__ err) {
  const int i = threadIdx.x;
  if (i >= n || i == skip) return;
  const long long t0 = clock64();
  for (;;) {
    int v;
    asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(flags + i) : "memory");
    if (v >= value) break;
    if (clock64() - t0 > (1ll << 32)) { atomicCAS(err, 0, kErrPeerWait); break; }     // ~2 s: a peer died
    __nanosleep(32);
  }
}

namespace ovn {

int sanitize_indices(ovn_handle* h, const int32_t* d_in, int n, int64_t limit, int code, int32_t* d_out, cudaStream_t s,
                     const int32_t* row_bad) {
  if (n <= 0) return OVN_OK;
  k_sanitize_idx<<<(n + 255) / 256, 256, 0, s>>>(d_in, d_out, n, limit < 1 ? 1 : limit, code, row_bad, h->d_err);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

// The caller has queued everything on `s`; this copies the flag back, synchronises `s` and maps a
// non-zero flag to a status (the flag is cleared so that the handle stays usable).
int check_device_error(ovn_handle* h, cudaStream_t s) {
  if (!h->h_pinned || !h->d_err) return OVN_OK;
  int32_t* hp = &h->stage()->err;
  OVN_CUDA(h, cudaMemcpyAsync(hp, h->d_err, sizeof(int), cudaMemcpyDeviceToHost, s));
  OVN_CUDA(h, cudaStreamSynchronize(s));
  const int e = *hp;
  if (e == 0) return OVN_OK;
  OVN_CUDA(h, cudaMemsetAsync(h->d_err, 0, sizeof(int), s));
  const char* ring = nullptr;          // a ring wait timed out: producer codes are 1xx, consumer codes 2xx / 4xx
  switch (e) {
    case kErrBadIndex: OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "a pair / candidate index is outside [0, bank_size)");
    case kErrIcpBadIndex:
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_icp_pairs: a scan index is outside [0, n_scans) (that pair's outputs "
                  "are poisoned: NaN pose, status OVN_ICP_BAD_INDEX)");
    case kErrRowNotPrepared:
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "resident bank: an indexed row was never passed to ovn_bank_prepare");
    case kErrNonFiniteOperand:
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "a value is not finite in the fp16 operands of the tensor-core path: a feature "
                  "volume given to the heads (NaN, inf, or |x - centre| > 65504; outputs of the call are poisoned, NaN / "
                  "INT32_MIN), or in the tensor-core leg an input pixel (NaN, inf) or an activation of s_conv1 .. the "
                  "last layer but one (above 65504; the feature volumes of the call are not valid)");
    case kErrPeerWait: OVN_SET_ERR(h, OVN_ERR_CUDA, "ovn_peer_wait timed out: a peer rank never signalled");
    case kErrInjectedFault: OVN_SET_ERR(h, OVN_ERR_CUDA, "tensor-core pipeline failed: k_conv2_wgmma: fault injected by "
                                        "OVN_DEBUG_FAULT (code %d); outputs of the call are poisoned (NaN / INT32_MIN)", e);
    case kErrDeltaLeftProducer: case kErrDeltaLeftConsumer: ring = "k_delta_conv1_wgmma: LEFT volume ring"; break;
    case kErrDeltaRightProducer: case kErrDeltaRightConsumer: ring = "k_delta_conv1_wgmma: RIGHT window ring"; break;
    case kErrDeltaW1Producer: case kErrDeltaW1Consumer: ring = "k_delta_conv1_wgmma: W1 ring"; break;
    case kErrDeltaO1Producer: case kErrDeltaO1Consumer: ring = "k_delta_conv1_wgmma: o1 staging"; break;
    case kErrConv2Producer: case kErrConv2Consumer: ring = "k_conv2_wgmma: o1 + W2 ring"; break;
    case kErrConv3X3Producer: case kErrConv3X3Consumer: ring = "k_conv3_wgmma: x3 ring"; break;
    case kErrConv3W3Producer: case kErrConv3W3Consumer: ring = "k_conv3_wgmma: W3 ring"; break;
    case kErrCorrRightProducer: case kErrCorrRightConsumer: ring = "k_corr_wgmma: RIGHT third ring"; break;
    case kErrCorrLeftProducer: case kErrCorrLeftConsumer: ring = "k_corr_wgmma: LEFT tile ring"; break;
  }
  if (!ring) OVN_SET_ERR(h, OVN_ERR_CUDA, "unknown device error code %d", e);
  OVN_SET_ERR(h, OVN_ERR_CUDA, "tensor-core pipeline failed: %s, %s wait timed out (code %d); outputs of the call are "
              "poisoned (NaN / INT32_MIN)", ring, e < 200 ? "producer" : "consumer", e);
}

}  // namespace ovn

extern "C" {

int ovn_abi_version(void) { return OVN_ABI_VERSION; }

const char* ovn_status_string(int status) {
  switch (status) {
    case OVN_OK: return "OVN_OK";
    case OVN_ERR_INVALID_ARG: return "OVN_ERR_INVALID_ARG";
    case OVN_ERR_BAD_CONFIG: return "OVN_ERR_BAD_CONFIG";
    case OVN_ERR_WEIGHTS: return "OVN_ERR_WEIGHTS";
    case OVN_ERR_CUDA: return "OVN_ERR_CUDA";
    case OVN_ERR_NO_DEVICE: return "OVN_ERR_NO_DEVICE";
    case OVN_ERR_CAPACITY: return "OVN_ERR_CAPACITY";
    default: return "OVN_ERR_UNKNOWN";
  }
}

void ovn_default_config(ovn_config* c) {
  if (!c) return;
  memset(c, 0, sizeof(*c));
  c->abi_version = OVN_ABI_VERSION;
  c->proj_H = 64; c->proj_W = 900;                 // config/network.yml:75
  c->fov_up_deg = 3.0f; c->fov_down_deg = -25.0f;  // utils.py:59
  c->max_range = 50.0f;
  c->use_depth = 1; c->use_normals = 1;            // network.yml:20-24
  c->n_prob_channels = 0; c->use_intensity = 0;
  c->strides_layer1[0] = 2; c->strides_layer1[1] = 2;   // network.yml:79
  c->additional_unsymmetric_layer3a = 1;           // network.yml:82
  c->leg_output_width = 360;                       // network.yml:77
  c->conv1size = 15;                               // generateNet.py:88-89
  c->precision = OVN_PREC_F16_TC;
  c->max_batch_scans = 16;                         // network.yml:41 batch_size
  c->max_batch_pairs = 1101;
}

static thread_local std::string g_create_error;

const char* ovn_last_error(const ovn_handle* h) { return h ? h->last_error.c_str() : g_create_error.c_str(); }
int64_t ovn_launch_count(const ovn_handle* h) { return h ? h->launches : 0; }
int ovn_input_channels(const ovn_handle* h) { return h ? h->C : 0; }
int ovn_feature_width(const ovn_handle* h) { return h ? h->cfg.leg_output_width : 0; }
int ovn_feature_channels(const ovn_handle* h) { return h ? kFeatC : 0; }

#define CREATE_FAIL(code, ...)                              \
  do {                                                      \
    char _b[512];                                           \
    snprintf(_b, sizeof(_b), __VA_ARGS__);                  \
    g_create_error = _b;                                    \
    return (code);                                          \
  } while (0)

// consumes the error like OVN_CUDA, so that it is reported once
#define CREATE_CUDA(call)                                                              \
  do {                                                                                 \
    cudaError_t _e = (call);                                                           \
    if (_e != cudaSuccess) {                                                           \
      cudaGetLastError();                                                              \
      CREATE_FAIL(OVN_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(_e));              \
    }                                                                                  \
  } while (0)

// a workspace allocation of ovn_create: its message is the one Buffer::ensure left in the handle
#define CREATE_ALLOC(buf, bytes)                                                       \
  do {                                                                                 \
    if ((buf).ensure(h.get(), (bytes)) != OVN_OK) CREATE_FAIL(OVN_ERR_CUDA, "ovn_create: %s", h->last_error.c_str()); \
  } while (0)

ovn_handle::~ovn_handle() {
  if (ev_bank) cudaEventDestroy(ev_bank);
  if (own_stream) cudaStreamDestroy(own_stream);
  for (auto& v : prof_ev) for (cudaEvent_t e : v) cudaEventDestroy(e);
}

int ovn_create(const ovn_config* cfg, ovn_handle** out) {
  if (!cfg || !out) CREATE_FAIL(OVN_ERR_INVALID_ARG, "ovn_create: NULL argument");
  *out = nullptr;
  if (cfg->abi_version != OVN_ABI_VERSION)
    CREATE_FAIL(OVN_ERR_INVALID_ARG, "ovn_create: abi_version %d != %d", cfg->abi_version, OVN_ABI_VERSION);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    CREATE_FAIL(OVN_ERR_NO_DEVICE, "ovn_create: no CUDA device visible (this library has no CPU fallback)");
  }
  int dev = 0;
  CREATE_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  CREATE_CUDA(cudaGetDeviceProperties(&prop, dev));
  if (prop.major != 9 || prop.minor != 0)
    CREATE_FAIL(OVN_ERR_NO_DEVICE, "ovn_create: device %d is sm_%d%d; this build targets sm_90a only", dev,
                prop.major, prop.minor);
  std::unique_ptr<ovn_handle> h(new ovn_handle());
  h->cfg = *cfg;
  h->device = dev;
  h->sm_count = prop.multiProcessorCount;
  const ovn_config& c = h->cfg;
  if (c.proj_H <= 0 || c.proj_W <= 0 || c.max_batch_scans <= 0 || c.max_batch_pairs <= 0)
    CREATE_FAIL(OVN_ERR_BAD_CONFIG, "ovn_create: non-positive size in config");
  if (c.n_prob_channels != 0 && c.n_prob_channels != 3 && c.n_prob_channels != 20)
    CREATE_FAIL(OVN_ERR_BAD_CONFIG, "ovn_create: n_prob_channels must be 0, 3 or 20 (infer.py:68-73)");
  h->C = (c.use_depth ? 1 : 0) + (c.use_normals ? 3 : 0) + c.n_prob_channels + (c.use_intensity ? 1 : 0);
  if (h->C <= 0) CREATE_FAIL(OVN_ERR_BAD_CONFIG, "ovn_create: no input channel enabled");

  // ---- leg shape inference (generateNet.py:161-217).  A config whose leg does not reduce the image
  // to 1 x leg_output_width x 128 still gets a handle, but only the projection stages work on it.
  struct { int kh, kw, sh, sw, cout; bool opt; } T[] = {
      {5, 15, c.strides_layer1[0], c.strides_layer1[1], 16, false}, {3, 15, 2, 1, 32, false},
      {3, 15, 2, 1, 64, false},  {3, 12, 2, 1, 64, true},           {2, 9, 2, 1, 128, false},
      {1, 9, 1, 1, 128, false},  {1, 9, 1, 1, 128, false},          {1, 9, 1, 1, 128, false},
      {1, 7, 1, 1, 128, false},  {1, 5, 1, 1, 128, false},          {1, 3, 1, 1, 128, false}};
  int hh = c.proj_H, ww = c.proj_W, cc = h->C;
  h->n_leg = 0;
  h->net_ok = true;
  char nb[256];
  for (int i = 0; i < 11 && h->net_ok; ++i) {
    if (T[i].opt && !c.additional_unsymmetric_layer3a) continue;
    if (T[i].sh <= 0 || T[i].sw <= 0 || hh < T[i].kh || ww < T[i].kw) {
      snprintf(nb, sizeof(nb), "layer %s does not fit its input %dx%d", kLegNames[i], hh, ww);
      h->net_ok = false; h->net_error = nb;
      break;
    }
    set_spec(h->leg[h->n_leg], kLegNames[i], T[i].kh, T[i].kw, T[i].sh, T[i].sw, cc, T[i].cout, 1, hh, ww);
    hh = h->leg[h->n_leg].h_out; ww = h->leg[h->n_leg].w_out; cc = T[i].cout;
    h->n_leg++;
  }
  const int Wf = c.leg_output_width, s = c.conv1size;
  if (h->net_ok && (hh != 1 || ww != c.leg_output_width || cc != kFeatC)) {
    snprintf(nb, sizeof(nb), "leg output is %dx%dx%d, expected 1x%dx%d (network.yml:77)", hh, ww, cc,
             c.leg_output_width, kFeatC);
    h->net_ok = false; h->net_error = nb;
  }
  if (h->net_ok && (s <= 0 || Wf % s != 0 || Wf / s < 3)) {
    snprintf(nb, sizeof(nb), "conv1size %d must divide leg_output_width %d", s, Wf);
    h->net_ok = false; h->net_error = nb;
  }
  if (!h->net_ok) { h->n_leg = 0; *out = nullptr; }
  // ---- head shapes (generateNet.py:96-114)
  if (h->net_ok) {
    set_spec(h->head[0], "c_conv1", 1, s, 1, s, kFeatC, 64, 0, Wf, Wf);
    set_spec(h->head[1], "c_conv2", s, 1, s, 1, 64, 128, 1, h->head[0].h_out, h->head[0].w_out);
    set_spec(h->head[2], "c_conv3", 3, 3, 1, 1, 128, 256, 1, h->head[1].h_out, h->head[1].w_out);
    h->o1_h = h->head[0].h_out; h->o1_w = h->head[0].w_out;
    h->o2_h = h->head[1].h_out; h->o2_w = h->head[1].w_out;
    h->o3_h = h->head[2].h_out; h->o3_w = h->head[2].w_out;
    h->dense_in = h->o3_h * h->o3_w * h->head[2].cout;
    ParamLayout& P = h->params;
    for (int i = 0; i < 4 + h->n_leg; ++i) {
      const int slot = flat_slot(i);
      int64_t nb;
      P.off[slot] = P.n_total;
      slot_sizes(h.get(), slot, &P.n_kernel[slot], &nb);
      P.n_total += P.n_kernel[slot] + nb;
      if (i == 3) P.n_head = P.n_total;
    }
  }

  // ---- workspaces
  const size_t HW = (size_t)c.proj_H * c.proj_W;
  const size_t maxp = c.max_batch_pairs;
  // a handle with probability channels keeps a second key image per scan for ovn_preprocess_cues_batch
  CREATE_ALLOC(h->d_keys, (c.n_prob_channels > 0 ? 2 : 1) * c.max_batch_scans * HW * sizeof(unsigned long long));
  CREATE_ALLOC(h->d_input, c.max_batch_scans * HW * h->C * sizeof(float));
  CREATE_ALLOC(h->d_query_fv, (size_t)Wf * kFeatC * sizeof(float));
  CREATE_ALLOC(h->d_cand_idx, maxp * sizeof(int32_t));
  CREATE_ALLOC(h->d_query_yaw, maxp * sizeof(int32_t));
  CREATE_ALLOC(h->d_idx_san, 3 * maxp * sizeof(int32_t));   // left, right, resident-row check
  CREATE_ALLOC(h->d_err, sizeof(int));
  CREATE_CUDA(cudaMemset(h->d_err, 0, sizeof(int)));
  CREATE_CUDA(cudaEventCreateWithFlags(&h->ev_bank, cudaEventDisableTiming));
  CREATE_ALLOC(h->h_pinned, sizeof(StageHeader) + maxp * 3 * sizeof(int32_t));
  CREATE_ALLOC(h->d_query_overlap, maxp * sizeof(float));
  if (c.precision == OVN_PREC_FP32 && h->net_ok) {
    size_t max_act = 0;
    for (int l = 0; l < h->n_leg; ++l) {
      const size_t a = (size_t)h->leg[l].h_out * h->leg[l].w_out * h->leg[l].cout;
      if (a > max_act) max_act = a;
    }
    CREATE_ALLOC(h->d_act[0], max_act * c.max_batch_scans * sizeof(float));
    CREATE_ALLOC(h->d_act[1], max_act * c.max_batch_scans * sizeof(float));
    CREATE_ALLOC(h->d_o1, maxp * h->o1_h * h->o1_w * 64 * sizeof(float));
    CREATE_ALLOC(h->d_o2, maxp * h->o2_h * h->o2_w * 128 * sizeof(float));
    CREATE_ALLOC(h->d_G, maxp * Wf * Wf * sizeof(float));
  } else if (c.precision != OVN_PREC_F16_TC && c.precision != OVN_PREC_FP32) {
    CREATE_FAIL(OVN_ERR_BAD_CONFIG, "ovn_create: unknown precision %d", c.precision);
  }
  CREATE_CUDA(cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking));
  *out = h.release();
  return OVN_OK;
}

int ovn_destroy(ovn_handle* h) {
  if (!h) return OVN_OK;
  DeviceGuard guard(h);
  if (!h->open_shards.empty() || !h->own_shards.empty()) {
    cudaDeviceSynchronize();               // no queued gather still reads a shard; then the mappings, then the own shards
    h->open_shards.clear();
    h->own_shards.clear();
  }
  delete h;
  return OVN_OK;
}

int ovn_profile_enable(ovn_handle* h, int on) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  h->profiling = on != 0;
  return OVN_OK;
}

int ovn_profile_read(ovn_handle* h, const char* kernel, double* total_ms, int64_t* launches) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  if (!kernel || !total_ms || !launches) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_profile_read: NULL argument");
  static const char* names[kProfKinds] = {"delta_conv1", "conv2", "conv3", "corr", "project_scatter",
                                          "project_gather", "leg", "gather_rows", "rows_topk", "pgo_graphs",
                                          "render_scatter", "render_gather", "surfel_build", "surfel_scatter",
                                          "surfel_gather"};
  int kind = -1;
  for (int i = 0; i < kProfKinds; ++i) if (strcmp(kernel, names[i]) == 0) kind = i;
  if (kind < 0) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_profile_read: unknown kernel '%s'", kernel);
  OVN_CUDA(h, cudaDeviceSynchronize());
  { int rc = check_device_error(h, h->own_stream); if (rc != OVN_OK) return rc; }
  std::vector<cudaEvent_t>& ev = h->prof_ev[kind];
  double ms = 0;
  int64_t n = 0;
  for (size_t i = 0; i + 1 < ev.size(); i += 2) {
    float t = 0;
    if (cudaEventElapsedTime(&t, ev[i], ev[i + 1]) == cudaSuccess) { ms += t; ++n; }
  }
  for (cudaEvent_t e : ev) cudaEventDestroy(e);
  ev.clear();
  *total_ms = ms;
  *launches = n;
  return OVN_OK;
}

// ---- weights ------------------------------------------------------------------------------------
static const ConvSpec* find_layer(const ovn_handle* h, const char* name, int* slot) {
  for (int l = 0; l < h->n_leg; ++l)
    if (strcmp(h->leg[l].name, name) == 0) { *slot = l; return &h->leg[l]; }
  for (int l = 0; l < 3; ++l)
    if (strcmp(h->head[l].name, name) == 0) { *slot = kMaxLegLayers + l; return &h->head[l]; }
  return nullptr;
}

int ovn_set_weights(ovn_handle* h, const char* name, const float* k, const int64_t* dims, int32_t ndim,
                    const float* bias, int64_t bias_len) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  if (!name || !k || !dims || !bias) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_set_weights: NULL argument");
  if (!h->net_ok) OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_set_weights: %s", h->net_error.c_str());
  int slot = -1;
  int64_t expect[4];
  int expect_nd = 0;
  int64_t expect_bias = 0;
  if (strcmp(name, "overlap_output") == 0) {
    expect[0] = h->dense_in; expect[1] = 1; expect_nd = 2; expect_bias = 1;
  } else {
    const ConvSpec* L = find_layer(h, name, &slot);
    if (!L) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "ovn_set_weights: unknown layer name '%s'", name);
    expect[0] = L->kh; expect[1] = L->kw; expect[2] = L->cin; expect[3] = L->cout; expect_nd = 4;
    expect_bias = L->cout;
  }
  if (ndim != expect_nd || bias_len != expect_bias)
    OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "ovn_set_weights: layer %s expects a %d-d kernel and %lld biases", name,
                expect_nd, (long long)expect_bias);
  int64_t total = 1;
  for (int i = 0; i < ndim; ++i) {
    if (dims[i] != expect[i])
      OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "ovn_set_weights: layer %s kernel dim %d is %lld, expected %lld", name, i,
                  (long long)dims[i], (long long)expect[i]);
    total *= dims[i];
  }
  LayerWeights& w = h->host_w[name];
  w.kernel.assign(k, k + total);
  w.dims.assign(dims, dims + ndim);
  w.bias.assign(bias, bias + bias_len);
  w.set = true;
  h->weights_ready = false;
  return OVN_OK;
}

static int upload(ovn_handle* h, int slot, const LayerWeights& w) {
  const int rc = upload_vec(h, h->d_w[slot], w.kernel);
  return rc != OVN_OK ? rc : upload_vec(h, h->d_b[slot], w.bias);
}

int ovn_finalize_weights(ovn_handle* h) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  if (!h->net_ok) OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_finalize_weights: %s", h->net_error.c_str());
  for (int l = 0; l < h->n_leg; ++l) {
    auto it = h->host_w.find(h->leg[l].name);
    if (it == h->host_w.end() || !it->second.set)
      OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "ovn_finalize_weights: layer %s has no weights", h->leg[l].name);
    int rc = upload(h, l, it->second);
    if (rc != OVN_OK) return rc;
  }
  const char* hn[4] = {"c_conv1", "c_conv2", "c_conv3", "overlap_output"};
  for (int l = 0; l < 4; ++l) {
    auto it = h->host_w.find(hn[l]);
    if (it == h->host_w.end() || !it->second.set)
      OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "ovn_finalize_weights: layer %s has no weights", hn[l]);
    int rc = upload(h, kMaxLegLayers + l, it->second);
    if (rc != OVN_OK) return rc;
  }
  if (h->cfg.precision == OVN_PREC_F16_TC) {
    int rc = tc_pack_weights(h);
    if (rc != OVN_OK) return rc;
  }
  if (h->train) {                        // new weights: Adagrad starts over, old gradients are stale
    OVN_CUDA(h, cudaMemset(h->train->accum, 0, (size_t)h->params.n_total * sizeof(float)));
    h->train->grads = kNoGrads;
  }
  h->weights_ready = true;
  return OVN_OK;
}

// kernel / bias sizes and weight slot of a layer; dense = overlap_output
static int layer_slot(const ovn_handle* h, const char* name, int64_t* n_kernel, int64_t* n_bias, bool* head) {
  int slot = kMaxLegLayers + 3;
  if (strcmp(name, "overlap_output") != 0 && !find_layer(h, name, &slot)) return -1;
  slot_sizes(h, slot, n_kernel, n_bias);
  *head = slot >= kMaxLegLayers;
  return slot;
}

int ovn_get_weights(ovn_handle* h, const char* name, float* h_kernel, float* h_bias) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  if (!name || !h_kernel || !h_bias) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_get_weights: NULL argument");
  if (!h->weights_ready) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "ovn_get_weights: weights not finalised");
  int64_t nk, nb;
  bool head;
  const int slot = layer_slot(h, name, &nk, &nb, &head);
  if (slot < 0) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "ovn_get_weights: unknown layer name '%s'", name);
  OVN_CUDA(h, cudaDeviceSynchronize());            // weights may be updated by work queued on any stream
  OVN_CUDA(h, cudaMemcpy(h_kernel, h->d_w[slot], nk * sizeof(float), cudaMemcpyDeviceToHost));
  OVN_CUDA(h, cudaMemcpy(h_bias, h->d_b[slot], nb * sizeof(float), cudaMemcpyDeviceToHost));
  return OVN_OK;
}

int ovn_get_gradients(ovn_handle* h, const char* name, float* h_kernel, float* h_bias) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  if (!name || !h_kernel || !h_bias) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_get_gradients: NULL argument");
  int64_t nk, nb;
  bool head;
  const int slot = layer_slot(h, name, &nk, &nb, &head);
  if (slot < 0) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_get_gradients: '%s' is not a layer of the network", name);
  if (!head && (!h->train || h->train->grads < kNetGrads))
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_get_gradients: no valid gradients of leg layer '%s' (call "
                "ovn_net_gradients first)", name);
  if (!h->train || h->train->grads < kHeadGrads)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_get_gradients: no valid gradients (call ovn_head_gradients first)");
  const float* g = h->train->grad + h->params.off[slot];
  OVN_CUDA(h, cudaDeviceSynchronize());
  OVN_CUDA(h, cudaMemcpy(h_kernel, g, nk * sizeof(float), cudaMemcpyDeviceToHost));
  OVN_CUDA(h, cudaMemcpy(h_bias, g + nk, nb * sizeof(float), cudaMemcpyDeviceToHost));
  return OVN_OK;
}

// ---- stage entry points ---------------------------------------------------------------------------
#define REQUIRE(h, cond, msg) \
  do { if (!(cond)) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: %s", __func__, msg); } while (0)

int ovn_project_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int32_t n_scans,
                      int64_t n_total, float max_range, float* d_range, float* d_vertex, float* d_intensity,
                      int32_t* d_idx, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_scans >= 0 && n_total >= 0, "negative size");
  REQUIRE(h, n_scans == 0 || d_offsets, "d_offsets is NULL");
  REQUIRE(h, n_total == 0 || d_points, "d_points is NULL");
  return project_batch(h, d_points, d_offsets, n_scans, n_total, max_range, d_range, d_vertex, d_intensity, d_idx,
                       (cudaStream_t)stream);
}

int ovn_normals_batch(ovn_handle* h, const float* d_range, const float* d_vertex, int32_t n_scans, float* d_normal,
                      void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_scans >= 0, "negative size");
  REQUIRE(h, n_scans == 0 || (d_range && d_vertex && d_normal), "NULL image pointer");
  return normals_batch(h, d_range, d_vertex, n_scans, d_normal, (cudaStream_t)stream);
}

int ovn_semantic_batch(ovn_handle* h, const int32_t* d_idx, const float* d_probs, const int64_t* d_offsets,
                       int32_t n_scans, int32_t n_classes, float* d_out, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_scans >= 0 && n_classes > 0, "bad size");
  REQUIRE(h, n_scans == 0 || (d_idx && d_probs && d_offsets && d_out), "NULL pointer");
  return semantic_batch(h, d_idx, d_probs, d_offsets, n_scans, n_classes, d_out, (cudaStream_t)stream);
}

int ovn_gt_range_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int32_t n_scans,
                       int64_t n_total, const double* d_pose_ref, const double* d_pose_cur_inv, float max_range,
                       float* d_range, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_scans >= 0 && n_total >= 0, "negative size");
  REQUIRE(h, n_scans == 0 || (d_offsets && d_range && (d_points || n_total == 0)), "NULL pointer");
  return gt_range_batch(h, d_points, d_offsets, n_scans, n_total, d_pose_ref, d_pose_cur_inv, max_range, d_range,
                        (cudaStream_t)stream);
}

int ovn_gt_overlap_count(ovn_handle* h, const float* d_ref_ranges, const float* d_cur_range, int32_t n_scans,
                         int32_t* d_counts, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_scans >= 0, "negative size");
  REQUIRE(h, d_cur_range && d_counts && (n_scans == 0 || d_ref_ranges), "NULL pointer");
  return gt_overlap_count(h, d_ref_ranges, d_cur_range, n_scans, d_counts, (cudaStream_t)stream);
}

int ovn_gt_scan_radius(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int32_t n_scans,
                       double* d_radius, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_scans >= 0, "negative size");
  REQUIRE(h, n_scans == 0 || (d_points && d_offsets && d_radius), "NULL pointer");
  return gt_scan_radius(h, d_points, d_offsets, n_scans, d_radius, (cudaStream_t)stream);
}

int ovn_gt_pairs_count(ovn_handle* h, const float* d_points, const int64_t* h_offsets, int32_t n_ref,
                       const double* d_pose_ref, const double* d_radius, const float* d_cur_range,
                       const double* d_pose_cur_inv, int32_t n_cur, float max_range, int32_t tile_cur,
                       int32_t tile_ref, int32_t* d_counts, int64_t ld_counts, int64_t* d_n_pruned, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_ref >= 0 && n_cur >= 0, "negative size");
  REQUIRE(h, ld_counts >= n_ref, "ld_counts < n_ref");
  REQUIRE(h, n_cur == 0 || d_counts, "NULL pointer");
  REQUIRE(h, n_cur == 0 || n_ref == 0 || (d_points && h_offsets && d_pose_ref && d_radius && d_cur_range && d_pose_cur_inv),
          "NULL pointer");
  for (int32_t i = 0; i < n_ref && n_cur > 0; ++i)
    REQUIRE(h, h_offsets[i] >= 0 && h_offsets[i] <= h_offsets[i + 1], "h_offsets must be non-negative and non-decreasing");
  return gt_pairs_count(h, d_points, h_offsets, n_ref, d_pose_ref, d_radius, d_cur_range, d_pose_cur_inv, n_cur,
                        max_range, tile_cur, tile_ref, d_counts, ld_counts, d_n_pruned, (cudaStream_t)stream);
}

int ovn_preprocess_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int32_t n_scans,
                         int64_t n_total, const float* d_probs, float* d_input, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_scans >= 0 && n_total >= 0, "negative size");
  REQUIRE(h, n_scans == 0 || (d_offsets && d_input), "NULL pointer");
  return preprocess_batch(h, d_points, d_offsets, n_scans, n_total, d_probs, d_input, (cudaStream_t)stream);
}

int ovn_preprocess_cues_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int32_t n_scans,
                              int64_t n_total, const float* d_probs, float* d_input, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_scans >= 0 && n_total >= 0, "negative size");
  REQUIRE(h, n_scans == 0 || (d_offsets && d_input), "NULL pointer");
  return preprocess_cues_batch(h, d_points, d_offsets, n_scans, n_total, d_probs, d_input, (cudaStream_t)stream);
}

int ovn_render_batch(ovn_handle* h, const float* d_points, const int64_t* h_offsets, int32_t n_clouds,
                     int32_t n_virtual, const int64_t* h_entry_offsets, const int32_t* h_entry_cloud,
                     const double* h_entry_pose, float max_range, float* d_range, float* d_vertex, float* d_intensity,
                     int32_t* d_winner, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_clouds >= 0 && n_virtual >= 0, "negative size");
  REQUIRE(h, n_virtual == 0 || (h_offsets && h_entry_offsets), "NULL pointer");
  REQUIRE(h, n_virtual == 0 || h_entry_offsets[n_virtual] == 0 || (h_entry_cloud && h_entry_pose), "NULL pointer");
  return render_batch(h, d_points, h_offsets, n_clouds, n_virtual, h_entry_offsets, h_entry_cloud, h_entry_pose,
                      max_range, d_range, d_vertex, d_intensity, d_winner, (cudaStream_t)stream);
}

int ovn_render_preprocess_batch(ovn_handle* h, const float* d_points, const int64_t* h_offsets, int32_t n_clouds,
                                int32_t n_virtual, const int64_t* h_entry_offsets, const int32_t* h_entry_cloud,
                                const double* h_entry_pose, float* d_input, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_clouds >= 0 && n_virtual >= 0, "negative size");
  REQUIRE(h, n_virtual == 0 || (h_offsets && h_entry_offsets && d_input), "NULL pointer");
  REQUIRE(h, n_virtual == 0 || h_entry_offsets[n_virtual] == 0 || (h_entry_cloud && h_entry_pose), "NULL pointer");
  return render_preprocess_batch(h, d_points, h_offsets, n_clouds, n_virtual, h_entry_offsets, h_entry_cloud,
                                 h_entry_pose, d_input, (cudaStream_t)stream);
}

void ovn_surfel_default_params(ovn_surfel_params* p) {
  if (!p) return;
  p->kappa = 1.0;
  p->c_min = 0.5;
  p->max_splat = 8;
}

static int check_surfel_params(ovn_handle* h, const ovn_surfel_params* p, const char* fn) {
  if (!p) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: NULL surfel parameters", fn);
  if (!(std::isfinite(p->kappa) && std::isfinite(p->c_min)))
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: kappa and c_min must be finite", fn);
  if (!(p->kappa > 0.0)) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: kappa must be > 0", fn);
  if (!(p->c_min > 0.0 && p->c_min <= 1.0)) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: c_min must be in (0, 1]", fn);
  if (p->max_splat < 0 || p->max_splat > OVN_SURFEL_MAX_SPLAT_LIMIT)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: max_splat must be in [0, %d]", fn, OVN_SURFEL_MAX_SPLAT_LIMIT);
  return OVN_OK;
}

int ovn_surfels_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int32_t n_clouds,
                      int64_t n_total, const ovn_surfel_params* params, float* d_surfels, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  int rc = check_surfel_params(h, params, __func__);
  if (rc != OVN_OK) return rc;
  REQUIRE(h, n_clouds >= 0 && n_total >= 0, "negative size");
  REQUIRE(h, n_clouds == 0 || (d_offsets && d_surfels), "NULL pointer");
  REQUIRE(h, n_total == 0 || d_points, "NULL pointer");
  return surfels_batch(h, d_points, d_offsets, n_clouds, n_total, *params, d_surfels, (cudaStream_t)stream);
}

int ovn_render_surfels_batch(ovn_handle* h, const float* d_surfels, int32_t n_clouds, const double* d_rays,
                             int32_t n_virtual, const int64_t* h_entry_offsets, const int32_t* h_entry_cloud,
                             const double* h_entry_pose, const ovn_surfel_params* params, float max_range,
                             float* d_range, float* d_vertex, float* d_intensity, int32_t* d_winner, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  int rc = check_surfel_params(h, params, __func__);
  if (rc != OVN_OK) return rc;
  REQUIRE(h, n_clouds >= 0 && n_virtual >= 0, "negative size");
  REQUIRE(h, n_virtual == 0 || h_entry_offsets, "NULL pointer");
  REQUIRE(h, n_virtual == 0 || h_entry_offsets[n_virtual] == 0 || (h_entry_cloud && h_entry_pose), "NULL pointer");
  return render_surfels_batch(h, d_surfels, n_clouds, d_rays, n_virtual, h_entry_offsets, h_entry_cloud,
                              h_entry_pose, *params, max_range, d_range, d_vertex, d_intensity, d_winner,
                              (cudaStream_t)stream);
}

int ovn_render_surfels_preprocess_batch(ovn_handle* h, const float* d_surfels, int32_t n_clouds, const double* d_rays,
                                        int32_t n_virtual, const int64_t* h_entry_offsets,
                                        const int32_t* h_entry_cloud, const double* h_entry_pose,
                                        const ovn_surfel_params* params, float* d_input, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  int rc = check_surfel_params(h, params, __func__);
  if (rc != OVN_OK) return rc;
  REQUIRE(h, n_clouds >= 0 && n_virtual >= 0, "negative size");
  REQUIRE(h, n_virtual == 0 || (h_entry_offsets && d_input), "NULL pointer");
  REQUIRE(h, n_virtual == 0 || h_entry_offsets[n_virtual] == 0 || (h_entry_cloud && h_entry_pose), "NULL pointer");
  return render_surfels_preprocess_batch(h, d_surfels, n_clouds, d_rays, n_virtual, h_entry_offsets, h_entry_cloud,
                                         h_entry_pose, *params, d_input, (cudaStream_t)stream);
}

int ovn_pack_input(ovn_handle* h, const float* d_depth, const float* d_normal, const float* d_prob,
                   const float* d_intensity, int32_t n_scans, float* d_input, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_scans >= 0, "negative size");
  REQUIRE(h, (d_depth != nullptr) == (h->cfg.use_depth != 0), "depth pointer does not match use_depth");
  REQUIRE(h, (d_normal != nullptr) == (h->cfg.use_normals != 0), "normal pointer does not match use_normals");
  REQUIRE(h, (d_prob != nullptr) == (h->cfg.n_prob_channels != 0), "prob pointer does not match n_prob_channels");
  REQUIRE(h, (d_intensity != nullptr) == (h->cfg.use_intensity != 0), "intensity pointer does not match use_intensity");
  return pack_input(h, d_depth, d_normal, d_prob, d_intensity, n_scans, d_input, (cudaStream_t)stream);
}

int ovn_leg_forward(ovn_handle* h, const float* d_input, int32_t n_scans, float* d_fv, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_scans >= 0, "negative size");
  if (n_scans == 0) return OVN_OK;
  REQUIRE(h, d_input && d_fv, "NULL pointer");
  if (!h->net_ok) OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_leg_forward: %s", h->net_error.c_str());
  if (!h->weights_ready) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "ovn_leg_forward: weights not finalised");
  const int Wf = h->cfg.leg_output_width;
  const size_t in_stride = (size_t)h->cfg.proj_H * h->cfg.proj_W * h->C;
  for (int s0 = 0; s0 < n_scans; s0 += h->cfg.max_batch_scans) {
    const int n = (n_scans - s0 < h->cfg.max_batch_scans) ? n_scans - s0 : h->cfg.max_batch_scans;
    int rc = (h->cfg.precision == OVN_PREC_F16_TC)
                 ? leg_forward_tc(h, d_input + s0 * in_stride, n, d_fv + (size_t)s0 * Wf * kFeatC, (cudaStream_t)stream)
                 : leg_forward_fp32(h, d_input + s0 * in_stride, n, d_fv + (size_t)s0 * Wf * kFeatC, (cudaStream_t)stream);
    if (rc != OVN_OK) return rc;
  }
  return OVN_OK;
}

static int heads_dispatch(ovn_handle* h, const float* d_bank, int64_t bank_size, const float* d_query,
                          const int32_t* d_left, const int32_t* d_right, int n, float* d_overlap, int32_t* d_yaw,
                          float* d_corr, cudaStream_t s) {
  if (!h->net_ok) OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "heads: %s", h->net_error.c_str());
  if (!h->weights_ready) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "heads: weights not finalised");
  if (bank_size <= 0) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "heads: bank_size must be positive");
  // Every index list is bounds-checked on the device (no host sync): out-of-range entries are clamped,
  // the error flag is raised, the finalize kernels poison the outputs and the next synchronising
  // entry point (ovn_check, *_host, ovn_profile_read) returns OVN_ERR_INVALID_ARG.
  const int maxp = h->cfg.max_batch_pairs;
  const int Wf = h->cfg.leg_output_width;
  for (int p0 = 0; p0 < n; p0 += maxp) {
    const int np = (n - p0 < maxp) ? n - p0 : maxp;
    int32_t* l = h->d_idx_san;
    int32_t* r = d_right ? h->d_idx_san + maxp : nullptr;
    int rc = sanitize_indices(h, d_left + p0, np, bank_size, kErrBadIndex, l, s);
    if (rc == OVN_OK && d_right) rc = sanitize_indices(h, d_right + p0, np, bank_size, kErrBadIndex, r, s);
    if (rc != OVN_OK) return rc;
    float* corr = d_corr ? d_corr + (size_t)p0 * Wf : nullptr;
    rc = (h->cfg.precision == OVN_PREC_F16_TC)
             ? heads_forward_tc(h, d_bank, d_query, l, r, np, d_overlap + p0, d_yaw + p0, corr, s)
             : heads_forward_fp32(h, d_bank, d_query, l, r, np, d_overlap + p0, d_yaw + p0, corr, s);
    if (rc != OVN_OK) return rc;
  }
  return OVN_OK;
}

int ovn_heads_forward(ovn_handle* h, const float* d_bank, int64_t bank_size, const int32_t* d_left,
                      const int32_t* d_right, int32_t n_pairs, float* d_overlap, int32_t* d_yaw, float* d_corr,
                      void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_pairs >= 0 && bank_size >= 0, "negative size");
  if (n_pairs == 0) return OVN_OK;
  REQUIRE(h, d_bank && d_left && d_right && d_overlap && d_yaw, "NULL pointer");
  return heads_dispatch(h, d_bank, bank_size, nullptr, d_left, d_right, n_pairs, d_overlap, d_yaw, d_corr,
                        (cudaStream_t)stream);
}

int ovn_heads_1vsN(ovn_handle* h, const float* d_bank, int64_t bank_size, const float* d_query,
                   const int32_t* d_cand_idx, int32_t n_cand, float* d_overlap, int32_t* d_yaw, float* d_corr,
                   void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_cand >= 0 && bank_size >= 0, "negative size");
  if (n_cand == 0) return OVN_OK;
  REQUIRE(h, d_bank && d_query && d_overlap && d_yaw, "NULL pointer");
  cudaStream_t s = (cudaStream_t)stream;
  if (d_cand_idx)
    return heads_dispatch(h, d_bank, bank_size, d_query, d_cand_idx, nullptr, n_cand, d_overlap, d_yaw, d_corr, s);
  REQUIRE(h, n_cand <= bank_size, "n_cand exceeds bank_size");
  // candidates 0..n-1 in chunks of the scratch capacity
  const int maxp = h->cfg.max_batch_pairs;
  for (int p0 = 0; p0 < n_cand; p0 += maxp) {
    const int np = (n_cand - p0 < maxp) ? n_cand - p0 : maxp;
    k_iota<<<(np + 255) / 256, 256, 0, s>>>(h->d_cand_idx, np, p0);
    OVN_LAUNCH_CHECK(h);
    int rc = heads_dispatch(h, d_bank, bank_size, d_query, h->d_cand_idx, nullptr,
                            np, d_overlap + p0, d_yaw + p0,
                            d_corr ? d_corr + (size_t)p0 * h->cfg.leg_output_width : nullptr, s);
    if (rc != OVN_OK) return rc;
  }
  return OVN_OK;
}

int ovn_heads_rows_vs_bank(ovn_handle* h, const float* d_bank, int64_t bank_size, int64_t row_lo, int64_t row_hi,
                           float* d_overlap, int32_t* d_yaw, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, bank_size >= 0 && row_lo >= 0 && row_lo <= row_hi && row_hi <= bank_size, "bad row range");
  if (row_lo == row_hi || bank_size == 0) return OVN_OK;
  REQUIRE(h, d_bank && d_overlap && d_yaw, "NULL pointer");
  REQUIRE(h, bank_size <= INT32_MAX, "bank too large");
  const size_t vol = (size_t)h->cfg.leg_output_width * kFeatC;
  for (int64_t i = row_lo; i < row_hi; ++i) {
    int rc = ovn_heads_1vsN(h, d_bank, bank_size, d_bank + (size_t)i * vol, nullptr, (int32_t)bank_size,
                            d_overlap + (size_t)(i - row_lo) * bank_size, d_yaw + (size_t)(i - row_lo) * bank_size,
                            nullptr, stream);
    if (rc != OVN_OK) return rc;
  }
  return OVN_OK;
}

int ovn_rows_topk(ovn_handle* h, const float* d_overlap, const int32_t* d_yaw, int64_t rows, int64_t stride,
                  const int32_t* h_n, int32_t k, float* d_top_overlap, int32_t* d_top_index, int32_t* d_top_yaw,
                  void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, k >= 1 && k <= kTopkMax, "k must be in [1, 32]");
  REQUIRE(h, rows >= 0 && stride >= 0 && stride <= INT32_MAX, "rows and stride must be in [0, 2^31)");
  if (rows == 0) return OVN_OK;
  REQUIRE(h, d_overlap && d_yaw && h_n && d_top_overlap && d_top_index && d_top_yaw, "NULL pointer");
  std::vector<int64_t> off((size_t)rows);
  for (int64_t r = 0; r < rows; ++r) {
    if (h_n[r] < 0 || h_n[r] > stride)
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_rows_topk: n[%lld] = %d is outside [0, stride = %lld]", (long long)r,
                  h_n[r], (long long)stride);
    off[(size_t)r] = r * stride;
  }
  return rows_topk(h, d_overlap, d_yaw, off.data(), h_n, rows, k, d_top_overlap, d_top_index, d_top_yaw,
                   (cudaStream_t)stream);
}

int ovn_heads_prefix_topk(ovn_handle* h, const float* d_bank, int64_t bank_size, int64_t row_lo, int64_t row_hi,
                          const int32_t* h_n_cand, int32_t k, float* d_top_overlap, int32_t* d_top_index,
                          int32_t* d_top_yaw, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, k >= 1 && k <= kTopkMax, "k must be in [1, 32]");
  REQUIRE(h, bank_size >= 0 && bank_size <= INT32_MAX && row_lo >= 0 && row_lo <= row_hi && row_hi <= bank_size,
          "bad row range");
  if (row_lo == row_hi) return OVN_OK;
  REQUIRE(h, d_bank && h_n_cand && d_top_overlap && d_top_index && d_top_yaw, "NULL pointer");
  const int64_t rows = row_hi - row_lo;
  for (int64_t r = 0; r < rows; ++r)
    if (h_n_cand[r] < 0 || h_n_cand[r] > bank_size || h_n_cand[r] > kTopkScratchPairs)
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_heads_prefix_topk: n_cand[%lld] = %d is outside [0, bank_size = %lld]",
                  (long long)r, h_n_cand[r], (long long)bank_size);
  if (!h->net_ok) OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_heads_prefix_topk: %s", h->net_error.c_str());
  if (!h->weights_ready) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "ovn_heads_prefix_topk: weights not finalised");
  int rc = h->d_topk_scratch.ensure(h, (size_t)kTopkScratchPairs * (sizeof(float) + sizeof(int32_t)));
  if (rc != OVN_OK) return rc;
  float* s_ov = reinterpret_cast<float*>(h->d_topk_scratch.get());
  int32_t* s_yaw = reinterpret_cast<int32_t*>(s_ov + kTopkScratchPairs);
  const size_t vol = (size_t)h->cfg.leg_output_width * kFeatC;
  cudaStream_t s = (cudaStream_t)stream;
  // Rows are scored into the scratch back to back.  When the next row does not fit, one k_rows_topk launch reduces
  // the rows the scratch holds (a "fill"), and the next fill reuses it in stream order.
  std::vector<int64_t> off;
  std::vector<int32_t> len;
  int64_t used = 0, first = 0;
  auto reduce_fill = [&]() -> int {
    const int rc2 = rows_topk(h, s_ov, s_yaw, off.data(), len.data(), (int64_t)off.size(), k,
                              d_top_overlap + first * k, d_top_index + first * k, d_top_yaw + first * k, s);
    first += (int64_t)off.size();
    off.clear();
    len.clear();
    used = 0;
    return rc2;
  };
  for (int64_t r = 0; r < rows; ++r) {
    const int32_t n = h_n_cand[r];
    if (used + n > kTopkScratchPairs || (int64_t)off.size() == kTopkRowsPerLaunch) {
      if ((rc = reduce_fill()) != OVN_OK) return rc;
    }
    if (n > 0) {
      rc = ovn_heads_1vsN(h, d_bank, bank_size, d_bank + (size_t)(row_lo + r) * vol, nullptr, n, s_ov + used,
                          s_yaw + used, nullptr, stream);
      if (rc != OVN_OK) return rc;
    }
    off.push_back(used);
    len.push_back(n);
    used += n;
  }
  return reduce_fill();
}

// ---- Monte Carlo localization -------------------------------------------------------------------------------
static bool finite_nonneg(const double* v, int n) {
  for (int i = 0; i < n; ++i)
    if (!(v[i] >= 0.0 && v[i] < INFINITY)) return false;
  return true;
}

int ovn_mcl_set_map(ovn_handle* h, const double* h_keyframes, int32_t n_keyframes, const int32_t* h_raster,
                    int32_t rows, int32_t cols, double x0, double y0, double cell) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, h_keyframes && h_raster, "NULL pointer");
  REQUIRE(h, n_keyframes >= 1 && n_keyframes <= kMcMaxKeyframes, "n_keyframes must be in [1, 2^24]");
  REQUIRE(h, rows >= 1 && cols >= 1 && (int64_t)rows * cols <= kMcMaxCells, "rows, cols >= 1 and rows cols <= 2^28");
  REQUIRE(h, cell > 0.0 && cell < INFINITY && std::isfinite(x0) && std::isfinite(y0), "cell > 0 and finite origin");
  for (int64_t i = 0; i < (int64_t)n_keyframes * 3; ++i)
    if (!std::isfinite(h_keyframes[i])) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_mcl_set_map: keyframe value %lld is not finite", (long long)i);
  for (int64_t i = 0; i < (int64_t)rows * cols; ++i)
    if (h_raster[i] < -1 || h_raster[i] >= n_keyframes)
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_mcl_set_map: raster cell %lld = %d is outside [-1, %d)", (long long)i,
                  h_raster[i], n_keyframes);
  McState& m = h->mcl;
  m.n = 0;                                   // the set referred to the old map
  m.pending = -1;
  m.stages = 0;
  OVN_CUDA(h, cudaDeviceSynchronize());      // no queued kernel still reads the old map
  int rc;
  m.map = McMap{};
  if ((rc = m.kf.ensure(h, (size_t)n_keyframes * 3 * sizeof(double))) != OVN_OK ||
      (rc = m.raster.ensure(h, (size_t)rows * cols * sizeof(int32_t))) != OVN_OK ||
      (rc = m.flags.ensure(h, (size_t)n_keyframes * sizeof(int32_t))) != OVN_OK ||
      (rc = m.slot.ensure(h, (size_t)n_keyframes * sizeof(int32_t))) != OVN_OK)
    return rc;
  OVN_CUDA(h, cudaMemcpy(m.kf, h_keyframes, (size_t)n_keyframes * 3 * sizeof(double), cudaMemcpyHostToDevice));
  OVN_CUDA(h, cudaMemcpy(m.raster, h_raster, (size_t)rows * cols * sizeof(int32_t), cudaMemcpyHostToDevice));
  m.map.K = n_keyframes;
  m.map.rows = rows;
  m.map.cols = cols;
  m.map.x0 = x0;
  m.map.y0 = y0;
  m.map.cell = cell;
  return OVN_OK;
}

int ovn_mcl_init(ovn_handle* h, int32_t mode, int32_t n, uint64_t seed, const double* h_pose, const double* h_sigma,
                 double init_radius, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, h->mcl.map.K > 0, "no map: call ovn_mcl_set_map first");
  REQUIRE(h, n >= 1 && n <= kMcMaxParticles, "n must be in [1, 2^24]");
  if (mode == OVN_MCL_INIT_GLOBAL) {
    REQUIRE(h, init_radius >= 0.0 && init_radius < INFINITY, "init_radius must be finite and >= 0");
  } else if (mode == OVN_MCL_INIT_POSE) {
    REQUIRE(h, h_pose && h_sigma, "NULL pointer");
    REQUIRE(h, std::isfinite(h_pose[0]) && std::isfinite(h_pose[1]) && std::isfinite(h_pose[2]), "pose not finite");
    REQUIRE(h, finite_nonneg(h_sigma, 3), "sigma must be finite and >= 0");
  } else {
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_mcl_init: mode %d is not an ovn_mcl_init_mode", mode);
  }
  return mcl_init(h, mode, n, seed, mode == OVN_MCL_INIT_POSE ? h_pose : nullptr,
                  mode == OVN_MCL_INIT_POSE ? h_sigma : nullptr, init_radius, (cudaStream_t)stream);
}

int ovn_mcl_predict(ovn_handle* h, const double* h_odom, const double* h_sigma, int32_t* d_touched,
                    int32_t* h_n_touched, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, h->mcl.n > 0, "no particles: call ovn_mcl_init first");
  REQUIRE(h, h_odom && h_sigma && d_touched && h_n_touched, "NULL pointer");
  REQUIRE(h, std::isfinite(h_odom[0]) && std::isfinite(h_odom[1]) && std::isfinite(h_odom[2]), "odometry not finite");
  REQUIRE(h, finite_nonneg(h_sigma, 3), "sigma must be finite and >= 0");
  return mcl_predict(h, h_odom, h_sigma, d_touched, h_n_touched, (cudaStream_t)stream);
}

int ovn_mcl_update(ovn_handle* h, const float* d_overlap, const int32_t* d_yaw, int32_t n, double sigma_overlap,
                   double sigma_yaw, double rho, ovn_mcl_estimate* h_est, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, h->mcl.n > 0, "no particles: call ovn_mcl_init first");
  REQUIRE(h, h->mcl.pending >= 0, "no predict awaits an update");
  if (n != h->mcl.pending)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_mcl_update: n = %d, but the last predict touched %d keyframes", n,
                h->mcl.pending);
  REQUIRE(h, h_est && (n == 0 || (d_overlap && d_yaw)), "NULL pointer");
  REQUIRE(h, sigma_overlap > 0.0 && sigma_overlap < INFINITY && sigma_yaw > 0.0 && sigma_yaw < INFINITY,
          "sigma_overlap and sigma_yaw must be finite and > 0");
  REQUIRE(h, rho >= 0.0 && rho <= 1.0, "rho must be in [0, 1]");
  return mcl_update(h, d_overlap, d_yaw, sigma_overlap, sigma_yaw, rho, h_est, (cudaStream_t)stream);
}

int ovn_mcl_copy_particles(ovn_handle* h, double* d_out, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, h->mcl.n > 0, "no particles: call ovn_mcl_init first");
  REQUIRE(h, d_out, "NULL pointer");
  return mcl_copy_particles(h, d_out, (cudaStream_t)stream);
}

int ovn_mcl_copy_stage(ovn_handle* h, int32_t stage, void* d_out, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, stage >= OVN_MCL_STAGE_MOTION && stage <= OVN_MCL_STAGE_SCALARS, "stage is not an ovn_mcl_stage");
  REQUIRE(h, d_out, "NULL pointer");
  const int need = stage <= OVN_MCL_STAGE_LOOKUP ? kMcHeldPredict
                   : stage <= OVN_MCL_STAGE_WEIGHTS || stage == OVN_MCL_STAGE_SCALARS ? kMcHeldUpdate
                                                                                      : kMcHeldResample;
  if (!(h->mcl.stages & need))
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_mcl_copy_stage: stage %d is not held (no %s since the last init)", stage,
                need == kMcHeldPredict ? "predict" : need == kMcHeldUpdate ? "update" : "update that resampled");
  return mcl_copy_stage(h, stage, d_out, (cudaStream_t)stream);
}

int ovn_mcl_philox(ovn_handle* h, uint64_t seed, const uint32_t* d_ctr, int32_t n, uint32_t* d_out, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n >= 0, "n must be >= 0");
  REQUIRE(h, n == 0 || (d_ctr && d_out), "NULL pointer");
  return mcl_philox(h, seed, d_ctr, n, d_out, (cudaStream_t)stream);
}

// ---- point-to-plane ICP of loop-closure pairs ----------------------------------------------------------------
void ovn_icp_default_params(ovn_icp_params* p) {
  if (!p) return;
  p->d_start = 2.0;
  p->d_end = 0.3;
  p->gamma = 0.8;
  p->cos_normal = 0.86602540378443865;      // cos 30 deg
  p->eps_rot = 1e-6;
  p->eps_trans = 1e-5;
  p->iterations = 30;
  p->min_inliers = 100;
}

int ovn_icp_pairs(ovn_handle* h, const float* d_vertex, const float* d_normal, int32_t n_scans, const int32_t* d_src,
                  const int32_t* d_dst, const double* d_init, int32_t np, const ovn_icp_params* params,
                  ovn_icp_result* d_out, int32_t* d_assoc, double* d_system, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, params, "NULL pointer");
  REQUIRE(h, np >= 0, "np must be >= 0");
  const ovn_icp_params& p = *params;
  REQUIRE(h, p.iterations >= 1 && p.iterations <= OVN_ICP_MAX_ITERATIONS_LIMIT, "iterations must be in [1, 200]");
  REQUIRE(h, p.min_inliers >= 0, "min_inliers must be >= 0");
  REQUIRE(h, std::isfinite(p.d_start) && std::isfinite(p.d_end) && std::isfinite(p.gamma) &&
                 std::isfinite(p.cos_normal) && std::isfinite(p.eps_rot) && std::isfinite(p.eps_trans),
          "every ICP parameter must be finite");
  REQUIRE(h, p.d_end > 0.0 && p.d_end <= p.d_start, "0 < d_end <= d_start");
  REQUIRE(h, p.gamma > 0.0 && p.gamma <= 1.0, "gamma must be in (0, 1]");
  REQUIRE(h, p.cos_normal >= 0.0 && p.cos_normal <= 1.0, "cos_normal must be in [0, 1]");
  REQUIRE(h, p.eps_rot >= 0.0 && p.eps_trans >= 0.0, "eps_rot and eps_trans must be >= 0");
  if (np == 0) return OVN_OK;
  REQUIRE(h, d_vertex && d_normal && d_src && d_dst && d_init && d_out, "NULL pointer");
  REQUIRE(h, n_scans >= 1, "n_scans must be >= 1");
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<double> init((size_t)np * 16);
  OVN_CUDA(h, cudaMemcpyAsync(init.data(), d_init, init.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  OVN_CUDA(h, cudaStreamSynchronize(s));
  for (size_t i = 0; i < init.size(); ++i)
    if (!std::isfinite(init[i]))
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_icp_pairs: d_init[%lld][%lld] is not finite", (long long)(i / 16),
                  (long long)(i % 16));
  return icp_pairs(h, d_vertex, d_normal, n_scans, d_src, d_dst, d_init, np, p, d_out, d_assoc, d_system, s);
}

// ---- robust pose-graph optimization (DESIGN section 7, "Pose-graph optimization") -------------------------------
void ovn_pgo_default_params(ovn_pgo_params* p) {
  if (!p) return;
  p->phi = 25.0;
  p->lambda0 = 1e-6;
  p->lambda_min = 1e-12;
  p->lambda_max = 1e12;
  p->rel_cost_tol = 1e-10;
  p->step_tol = 1e-10;
  p->cg_tol = 1e-12;
  p->max_iterations = 50;
  p->max_cg_iterations = 2000;
}

// a finite row-major 4x4 whose bottom row is 0 0 0 1
static bool rigid_rows(const double* T) {
  for (int i = 0; i < 16; ++i)
    if (!std::isfinite(T[i])) return false;
  return T[12] == 0.0 && T[13] == 0.0 && T[14] == 0.0 && T[15] == 1.0;
}

int ovn_pgo_optimize_host(ovn_handle* h, int32_t n_graphs, const int64_t* node_offset, const int64_t* edge_offset,
                          const double* poses, const int32_t* edge_nodes, const double* edge_pose,
                          const double* edge_weight, const ovn_pgo_params* params, double* out_poses,
                          ovn_pgo_result* out_result, double* out_chi2, double* out_scale, double* out_gradient,
                          ovn_pgo_trial* out_trace, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  h->pgo_node_off.clear();      // pgo_graphs records the call again when it succeeds
  DeviceGuard guard(h);
  REQUIRE(h, params && node_offset && edge_offset && poses && edge_nodes && edge_pose && edge_weight && out_poses &&
                 out_result && out_chi2 && out_scale, "NULL pointer");
  REQUIRE(h, n_graphs >= 1 && n_graphs <= OVN_PGO_MAX_GRAPHS, "n_graphs must be in [1, 65535]");
  const ovn_pgo_params& p = *params;
  REQUIRE(h, p.phi > 0.0 && !std::isnan(p.phi), "phi must be > 0 (+inf: plain least squares)");
  REQUIRE(h, std::isfinite(p.lambda0) && std::isfinite(p.lambda_min) && std::isfinite(p.lambda_max) &&
                 p.lambda_min > 0.0 && p.lambda_min <= p.lambda0 && p.lambda0 <= p.lambda_max,
          "0 < lambda_min <= lambda0 <= lambda_max, all finite");
  REQUIRE(h, std::isfinite(p.rel_cost_tol) && std::isfinite(p.step_tol) && std::isfinite(p.cg_tol) &&
                 p.rel_cost_tol >= 0.0 && p.step_tol >= 0.0 && p.cg_tol >= 0.0,
          "rel_cost_tol, step_tol and cg_tol must be finite and >= 0");
  REQUIRE(h, p.max_iterations >= 0 && p.max_iterations <= OVN_PGO_MAX_ITERATIONS_LIMIT,
          "max_iterations must be in [0, 1000]");
  REQUIRE(h, p.max_cg_iterations >= 1 && p.max_cg_iterations <= OVN_PGO_MAX_CG_ITERATIONS_LIMIT,
          "max_cg_iterations must be in [1, 10000]");
  REQUIRE(h, node_offset[0] == 0 && edge_offset[0] == 0, "node_offset[0] and edge_offset[0] must be 0");
  for (int g = 0; g < n_graphs; ++g) {
    const int64_t n = node_offset[g + 1] - node_offset[g], ne = edge_offset[g + 1] - edge_offset[g];
    if (n < 2 || n > OVN_PGO_MAX_NODES)
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_pgo_optimize_host: graph %d has %lld nodes (2 .. %d)", g, (long long)n,
                  OVN_PGO_MAX_NODES);
    if (ne < n - 1 || ne > OVN_PGO_MAX_EDGES)
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_pgo_optimize_host: graph %d has %lld edges (n - 1 .. %d)", g,
                  (long long)ne, OVN_PGO_MAX_EDGES);
    for (int64_t i = node_offset[g]; i < node_offset[g + 1]; ++i)
      if (!rigid_rows(poses + 16 * i))
        OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_pgo_optimize_host: pose %lld of graph %d is not finite or its bottom "
                    "row is not 0 0 0 1", (long long)(i - node_offset[g]), g);
    for (int64_t k = edge_offset[g]; k < edge_offset[g + 1]; ++k) {
      const int64_t l = k - edge_offset[g];
      const int32_t a = edge_nodes[2 * k], b = edge_nodes[2 * k + 1];
      if (l < n - 1 && (a != l || b != l + 1))
        OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_pgo_optimize_host: edge %lld of graph %d is (%d, %d), but the first "
                    "n - 1 edges are the chain (k, k + 1)", (long long)l, g, a, b);
      if (a < 0 || a >= n || b < 0 || b >= n || a == b)
        OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_pgo_optimize_host: edge %lld of graph %d is (%d, %d): a node is "
                    "outside [0, %lld) or a == b", (long long)l, g, a, b, (long long)n);
      if (!rigid_rows(edge_pose + 16 * k))
        OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_pgo_optimize_host: the measurement of edge %lld of graph %d is not "
                    "finite or its bottom row is not 0 0 0 1", (long long)l, g);
      for (int t = 0; t < 6; ++t)
        if (!(std::isfinite(edge_weight[6 * k + t]) && edge_weight[6 * k + t] > 0.0))
          OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_pgo_optimize_host: weight %d of edge %lld of graph %d is not finite "
                      "and > 0", t, (long long)l, g);
    }
  }
  return pgo_graphs(h, n_graphs, node_offset, edge_offset, poses, edge_nodes, edge_pose, edge_weight, p, out_poses,
                    out_result, out_chi2, out_scale, out_gradient, out_trace, (cudaStream_t)stream);
}

int ovn_pgo_copy_workspace(ovn_handle* h, int32_t array, int32_t graph, double* h_out) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, !h->pgo_node_off.empty(), "no successful ovn_pgo_optimize_host call since the last refused or failed one");
  REQUIRE(h, array >= OVN_PGO_T && array <= OVN_PGO_Y, "array is not an ovn_pgo_array");
  REQUIRE(h, graph >= 0 && graph + 1 < (int64_t)h->pgo_node_off.size(), "graph is not a graph of the last call");
  REQUIRE(h, h_out, "NULL pointer");
  return pgo_copy_workspace(h, array, graph, h_out);
}

// ---- training precision ---------------------------------------------------------------------------
int ovn_set_train_precision(ovn_handle* h, int32_t train_precision) {
  if (!h) return OVN_ERR_INVALID_ARG;
  if (h->cfg.precision != OVN_PREC_FP32)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_set_train_precision: training needs a precision fp32 handle");
  if (train_precision != OVN_TRAIN_FP32 && train_precision != OVN_TRAIN_TF32X3)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_set_train_precision: unknown training precision %d (0: fp32, 1: tf32x3)",
                train_precision);
  h->train_precision = train_precision;
  return OVN_OK;
}

// The two gradient calls run their products at the handle's training precision; every other entry point, and
// every return path of these two, leaves h->train_tc false.
struct TrainPrecisionScope {
  ovn_handle* h;
  explicit TrainPrecisionScope(ovn_handle* hh) : h(hh) { h->train_tc = h->train_precision == OVN_TRAIN_TF32X3; }
  ~TrainPrecisionScope() { h->train_tc = false; }
};

// ---- training: the overlap head with a frozen leg, or the whole network (360OutputkLegs) ---------------------
// What ovn_head_gradients (rows: the feature-volume bank) and ovn_net_gradients (rows: the image set), and their
// _chunks forms, share: the checks, the training state, both index lists bounds-checked against the n_rows rows,
// and after the flow's own work (`run`) the losses and the device error flag.  `ch` with grad NULL is a one-chunk
// call into the handle's gradients; else the chunks of a _chunks call, whose parts and losses go to the caller.
}  // extern "C"
template <class Run>
static int gradients_call(ovn_handle* h, bool whole_network, const char* fn, const float* d_rows, int64_t n_rows,
                          const int32_t* d_left_idx, const int32_t* d_right_idx, int32_t n_pairs,
                          const float* d_gt_overlap, const int32_t* d_gt_orientation, GradChunks& ch, float* h_loss,
                          cudaStream_t s, Run run) {
  const bool chunked = ch.grad != nullptr;
  if (!h->net_ok) OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "%s: %s", fn, h->net_error.c_str());
  if (h->cfg.precision != OVN_PREC_FP32)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "%s: training needs a precision fp32 handle", fn);
  if (!h->weights_ready) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "%s: weights not finalised", fn);
  if (n_pairs <= 0 || n_rows <= 0)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: n_pairs and %s must be positive", fn,
                whole_network ? "n_images" : "bank_size");
  if (!(d_rows && d_left_idx && d_right_idx && d_gt_overlap && d_gt_orientation && h_loss))
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: NULL pointer", fn);
  const int maxp = h->cfg.max_batch_pairs;
  if (n_pairs > maxp) OVN_SET_ERR(h, OVN_ERR_CAPACITY, "%s: n_pairs=%d exceeds max_batch_pairs=%d", fn, n_pairs, maxp);
  if (whole_network && n_pairs > net_max_pairs(h))
    OVN_SET_ERR(h, OVN_ERR_CAPACITY, "%s: n_pairs=%d exceeds the %d pairs one call can launch", fn, n_pairs,
                net_max_pairs(h));
  if (!h->train) {
    int rc = train_alloc(h);
    if (rc != OVN_OK) return rc;
  }
  TrainState& t = *h->train;
  t.grads = kNoGrads;
  t.stage_np = 0;
  t.stopped = false;
  struct ConsumeStop {                       // the stop applies to this one call, whatever it returns
    TrainState& t;
    ~ConsumeStop() { t.stop_stage = t.stop_layer = -1; }
  } consume{t};
  float* p_loss = h->stage()->loss;
  if (chunked) {
    const size_t bytes = (size_t)kMaxSumParts * 3 * sizeof(float);
    int rc = t.chunk_loss.ensure(h, bytes);
    if (rc == OVN_OK) rc = t.chunk_loss_host.ensure(h, bytes);
    if (rc != OVN_OK) return rc;
    ch.loss = t.chunk_loss;
    p_loss = t.chunk_loss_host;
    for (int c = 0; c < ch.n; ++c) {         // an empty chunk: a zero part and zero losses
      if (ch.size(c) > 0) continue;
      OVN_CUDA(h, cudaMemsetAsync(ch.grad + c * ch.stride, 0, (size_t)ch.stride * sizeof(float), s));
      OVN_CUDA(h, cudaMemsetAsync(ch.loss + 3 * c, 0, 3 * sizeof(float), s));
    }
  } else {
    ch.n = 1;
    ch.off[0] = 0;
    ch.off[1] = n_pairs;
    ch.grad = t.grad;
    ch.loss = t.loss;
  }
  int32_t* l = h->d_idx_san;
  int32_t* r = h->d_idx_san + maxp;
  int rc = sanitize_indices(h, d_left_idx, n_pairs, n_rows, kErrBadIndex, l, s);
  if (rc == OVN_OK) rc = sanitize_indices(h, d_right_idx, n_pairs, n_rows, kErrBadIndex, r, s);
  if (rc == OVN_OK) rc = run(l, r);
  if (rc != OVN_OK) return rc;
  if (!t.stopped)
    OVN_CUDA(h, cudaMemcpyAsync(p_loss, ch.loss, (size_t)ch.n * 3 * sizeof(float), cudaMemcpyDeviceToHost, s));
  rc = check_device_error(h, s);            // synchronises s; a bad index -> OVN_ERR_INVALID_ARG
  if (rc != OVN_OK) return rc;
  t.stage_np = n_pairs;
  t.stage_net = whole_network;
  t.stage_stop = t.stopped ? t.stop_stage : -1;
  t.stage_stop_layer = t.stopped ? t.stop_layer : -1;
  if (t.stopped) return OVN_OK;             // no losses, no gradients, no batch
  memcpy(h_loss, p_loss, (size_t)ch.n * 3 * sizeof(float));
  if (!chunked) t.grads = whole_network ? kNetGrads : kHeadGrads;
  return OVN_OK;
}

// The chunk table of a _chunks call: 1 <= n_chunks <= 64, offsets non-decreasing from 0 to n_pairs, parts of
// ovn_train_gradient_size floats each
static int chunk_table(ovn_handle* h, const char* fn, bool whole_network, int32_t n_pairs,
                       const int32_t* h_chunk_offsets, int32_t n_chunks, float* d_parts, GradChunks* ch) {
  if (n_chunks < 1) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: n_chunks must be at least 1", fn);
  if (n_chunks > kMaxSumParts)
    OVN_SET_ERR(h, OVN_ERR_CAPACITY, "%s: n_chunks=%d exceeds %d", fn, n_chunks, kMaxSumParts);
  if (!h_chunk_offsets || !d_parts) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: NULL pointer", fn);
  if (h_chunk_offsets[0] != 0 || h_chunk_offsets[n_chunks] != n_pairs)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: the chunk offsets must run from 0 to n_pairs=%d (got %d .. %d)", fn,
                n_pairs, h_chunk_offsets[0], h_chunk_offsets[n_chunks]);
  for (int c = 0; c < n_chunks; ++c)
    if (h_chunk_offsets[c + 1] < h_chunk_offsets[c])
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: chunk offset %d (%d) is below offset %d (%d)", fn, c + 1,
                  h_chunk_offsets[c + 1], c, h_chunk_offsets[c]);
  ch->n = n_chunks;
  for (int c = 0; c <= n_chunks; ++c) ch->off[c] = h_chunk_offsets[c];
  ch->grad = d_parts;
  ch->stride = whole_network ? h->params.n_total : h->params.n_head;
  return OVN_OK;
}
extern "C" {

int ovn_head_gradients(ovn_handle* h, const float* d_bank, int64_t bank_size, const int32_t* d_left_idx,
                       const int32_t* d_right_idx, int32_t n_pairs, const float* d_gt_overlap,
                       const int32_t* d_gt_orientation, float min_overlap_for_angle, float* h_loss, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  TrainPrecisionScope precision(h);
  cudaStream_t s = (cudaStream_t)stream;
  GradChunks ch;
  return gradients_call(h, false, "ovn_head_gradients", d_bank, bank_size, d_left_idx, d_right_idx, n_pairs,
                        d_gt_overlap, d_gt_orientation, ch, h_loss, s, [&](const int32_t* l, const int32_t* r) {
                          return head_gradients_fp32(h, d_bank, l, r, n_pairs, d_gt_overlap, d_gt_orientation,
                                                     min_overlap_for_angle, ch, s);
                        });
}

int ovn_net_gradients(ovn_handle* h, const float* d_images, int64_t n_images, const int32_t* d_left_idx,
                      const int32_t* d_right_idx, int32_t n_pairs, const float* d_gt_overlap,
                      const int32_t* d_gt_orientation, float min_overlap_for_angle, float* h_loss, float* d_fv_grad,
                      void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  TrainPrecisionScope precision(h);
  cudaStream_t s = (cudaStream_t)stream;
  GradChunks ch;
  return gradients_call(h, true, "ovn_net_gradients", d_images, n_images, d_left_idx, d_right_idx, n_pairs,
                        d_gt_overlap, d_gt_orientation, ch, h_loss, s, [&](const int32_t* l, const int32_t* r) {
                          return net_gradients_fp32(h, d_images, l, r, n_pairs, d_gt_overlap, d_gt_orientation,
                                                    min_overlap_for_angle, d_fv_grad, ch, s);
                        });
}

int ovn_head_gradients_chunks(ovn_handle* h, const float* d_bank, int64_t bank_size, const int32_t* d_left_idx,
                              const int32_t* d_right_idx, int32_t n_pairs, const int32_t* h_chunk_offsets,
                              int32_t n_chunks, const float* d_gt_overlap, const int32_t* d_gt_orientation,
                              float min_overlap_for_angle, float* d_parts, float* h_loss, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  TrainPrecisionScope precision(h);
  cudaStream_t s = (cudaStream_t)stream;
  const char* fn = "ovn_head_gradients_chunks";
  GradChunks ch;
  int rc = chunk_table(h, fn, false, n_pairs, h_chunk_offsets, n_chunks, d_parts, &ch);
  if (rc != OVN_OK) return rc;
  return gradients_call(h, false, fn, d_bank, bank_size, d_left_idx, d_right_idx, n_pairs, d_gt_overlap,
                        d_gt_orientation, ch, h_loss, s, [&](const int32_t* l, const int32_t* r) {
                          return head_gradients_fp32(h, d_bank, l, r, n_pairs, d_gt_overlap, d_gt_orientation,
                                                     min_overlap_for_angle, ch, s);
                        });
}

int ovn_net_gradients_chunks(ovn_handle* h, const float* d_images, int64_t n_images, const int32_t* d_left_idx,
                             const int32_t* d_right_idx, int32_t n_pairs, const int32_t* h_chunk_offsets,
                             int32_t n_chunks, const float* d_gt_overlap, const int32_t* d_gt_orientation,
                             float min_overlap_for_angle, float* d_parts, float* h_loss, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  TrainPrecisionScope precision(h);
  cudaStream_t s = (cudaStream_t)stream;
  const char* fn = "ovn_net_gradients_chunks";
  GradChunks ch;
  int rc = chunk_table(h, fn, true, n_pairs, h_chunk_offsets, n_chunks, d_parts, &ch);
  if (rc != OVN_OK) return rc;
  return gradients_call(h, true, fn, d_images, n_images, d_left_idx, d_right_idx, n_pairs, d_gt_overlap,
                        d_gt_orientation, ch, h_loss, s, [&](const int32_t* l, const int32_t* r) {
                          return net_gradients_fp32(h, d_images, l, r, n_pairs, d_gt_overlap, d_gt_orientation,
                                                    min_overlap_for_angle, nullptr, ch, s);
                        });
}

// ovn_head_adagrad_step / ovn_net_adagrad_step: the handle's own gradients as one part of weight 1
static int adagrad_step(ovn_handle* h, bool whole_network, float learning_rate, void* stream) {
  const char* fn = whole_network ? "ovn_net_adagrad_step" : "ovn_head_adagrad_step";
  DeviceGuard guard(h);
  if (h->cfg.precision != OVN_PREC_FP32)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "%s: training needs a precision fp32 handle", fn);
  if (!h->train || h->train->grads < (whole_network ? kNetGrads : kHeadGrads))
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: %s", fn,
                whole_network ? "no valid whole-network gradients (call ovn_net_gradients first)"
                              : "no valid gradients (call ovn_head_gradients first)");
  const float one = 1.f;
  return adagrad_sum_fp32(h, whole_network, h->train->grad, 1, &one, learning_rate, (cudaStream_t)stream);
}

int ovn_head_adagrad_step(ovn_handle* h, float learning_rate, void* stream) {
  return h ? adagrad_step(h, false, learning_rate, stream) : OVN_ERR_INVALID_ARG;
}

int ovn_net_adagrad_step(ovn_handle* h, float learning_rate, void* stream) {
  return h ? adagrad_step(h, true, learning_rate, stream) : OVN_ERR_INVALID_ARG;
}

// ---- data-parallel training ---------------------------------------------------------------------------------
int ovn_train_gradient_size(ovn_handle* h, int32_t whole_network, int64_t* n) {
  if (!h) return OVN_ERR_INVALID_ARG;
  REQUIRE(h, n, "NULL pointer");
  if (!h->net_ok) OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_train_gradient_size: %s", h->net_error.c_str());
  *n = whole_network ? h->params.n_total : h->params.n_head;
  return OVN_OK;
}

int ovn_copy_gradients(ovn_handle* h, int32_t whole_network, float* d_out, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  if (h->cfg.precision != OVN_PREC_FP32)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_copy_gradients: training needs a precision fp32 handle");
  REQUIRE(h, d_out, "NULL pointer");
  if (!h->train || h->train->grads < kHeadGrads)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_copy_gradients: no valid gradients (call ovn_head_gradients or "
                "ovn_net_gradients first)");
  if (whole_network && h->train->grads < kNetGrads)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_copy_gradients: no valid whole-network gradients (call "
                "ovn_net_gradients first)");
  const int64_t n = whole_network ? h->params.n_total : h->params.n_head;
  OVN_CUDA(h, cudaMemcpyAsync(d_out, h->train->grad, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice,
                              (cudaStream_t)stream));
  return OVN_OK;
}

int ovn_copy_net_volumes(ovn_handle* h, float* d_out, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  if (h->cfg.precision != OVN_PREC_FP32)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_copy_net_volumes: training needs a precision fp32 handle");
  REQUIRE(h, d_out, "NULL pointer");
  if (!h->train || h->train->grads < kNetGrads)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_copy_net_volumes: no valid whole-network batch (call ovn_net_gradients "
                "first)");
  return copy_net_volumes_fp32(h, d_out, (cudaStream_t)stream);
}

// ---- stages of a gradient call (tests and diagnostics) ------------------------------------------------------
static bool stop_stage(int32_t stage) { return stage >= OVN_TRAIN_STAGE_O1 && stage <= OVN_TRAIN_STAGE_LEG_DY; }
static bool layer_stage(int32_t stage) { return stage == OVN_TRAIN_STAGE_LEG_DY || stage == OVN_TRAIN_STAGE_ACT; }
static bool net_stage(int32_t stage) {
  return stage == OVN_TRAIN_STAGE_DFV_CORR || stage == OVN_TRAIN_STAGE_LEG_DY || stage >= OVN_TRAIN_STAGE_DCORR;
}

// A stage and layer the handle's network has: OVN_ERR_INVALID_ARG otherwise
static int check_train_stage(ovn_handle* h, const char* fn, int32_t stage, int32_t layer) {
  if (h->cfg.precision != OVN_PREC_FP32)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "%s: training needs a precision fp32 handle", fn);
  if (!h->net_ok) OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "%s: %s", fn, h->net_error.c_str());
  if (stage < OVN_TRAIN_STAGE_O1 || stage > OVN_TRAIN_STAGE_ACT)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: unknown ovn_train_stage %d", fn, stage);
  if (layer_stage(stage) ? (layer < 0 || layer >= h->n_leg) : layer != 0)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: layer %d of stage %d (a leg layer 0..%d for LEG_DY and ACT, else 0)", fn,
                layer, stage, h->n_leg - 1);
  return OVN_OK;
}

int ovn_set_train_stop(ovn_handle* h, int32_t stage, int32_t layer) {
  if (!h) return OVN_ERR_INVALID_ARG;
  const char* fn = "ovn_set_train_stop";
  if (stage != -1) {
    int rc = check_train_stage(h, fn, stage, layer);
    if (rc != OVN_OK) return rc;
    if (!stop_stage(stage))
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: stage %d is read after a whole call, not a stop", fn, stage);
  }
  if (!h->train) {
    int rc = train_alloc(h);
    if (rc != OVN_OK) return rc;
  }
  h->train->stop_stage = stage;
  h->train->stop_layer = stage == -1 ? -1 : layer;
  return OVN_OK;
}

// The stage is held when the last gradient call succeeded, ran the flow the stage belongs to and stopped at it (a
// stop stage) or ran to the end (any other stage)
static int held_stage(ovn_handle* h, const char* fn, int32_t stage, int32_t layer) {
  int rc = check_train_stage(h, fn, stage, layer);
  if (rc != OVN_OK) return rc;
  const TrainState* t = h->train.get();
  if (!t || t->stage_np == 0)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: no stages (no successful gradient call since the handle trained last)",
                fn);
  if (net_stage(stage) && !t->stage_net)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: stage %d exists after a whole-network call only", fn, stage);
  if (stop_stage(stage) ? (t->stage_stop != stage || t->stage_stop_layer != layer) : t->stage_stop != -1)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: stage %d layer %d is not held (the last call stopped at stage %d layer %d)",
                fn, stage, layer, t->stage_stop, t->stage_stop_layer);
  return OVN_OK;
}

int ovn_train_stage_size(ovn_handle* h, int32_t stage, int32_t layer, int64_t* n) {
  if (!h) return OVN_ERR_INVALID_ARG;
  REQUIRE(h, n, "NULL pointer");
  int rc = held_stage(h, "ovn_train_stage_size", stage, layer);
  if (rc != OVN_OK) return rc;
  *n = train_stage_floats(h, stage, layer);
  return OVN_OK;
}

int ovn_copy_train_stage(ovn_handle* h, int32_t stage, int32_t layer, float* d_out, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, d_out, "NULL pointer");
  int rc = held_stage(h, "ovn_copy_train_stage", stage, layer);
  if (rc != OVN_OK) return rc;
  return copy_train_stage_fp32(h, stage, layer, d_out, (cudaStream_t)stream);
}

// ovn_copy_train_state / ovn_set_train_state: the Adagrad accumulators, in the layout of ovn_copy_gradients
static int train_state_call(ovn_handle* h, const char* fn, const void* ptr) {
  if (!h->net_ok) OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "%s: %s", fn, h->net_error.c_str());
  if (h->cfg.precision != OVN_PREC_FP32)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "%s: training needs a precision fp32 handle", fn);
  if (!ptr) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: NULL pointer", fn);
  if (!h->weights_ready) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "%s: weights not finalised", fn);
  return OVN_OK;
}

int ovn_copy_train_state(ovn_handle* h, int32_t whole_network, float* d_out, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  int rc = train_state_call(h, "ovn_copy_train_state", d_out);
  if (rc != OVN_OK) return rc;
  const size_t bytes = (size_t)(whole_network ? h->params.n_total : h->params.n_head) * sizeof(float);
  if (!h->train) {                         // never trained: the accumulators Adagrad would start from
    OVN_CUDA(h, cudaMemsetAsync(d_out, 0, bytes, (cudaStream_t)stream));
    return OVN_OK;
  }
  OVN_CUDA(h, cudaMemcpyAsync(d_out, h->train->accum, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return OVN_OK;
}

int ovn_set_train_state(ovn_handle* h, int32_t whole_network, const float* d_in, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  int rc = train_state_call(h, "ovn_set_train_state", d_in);
  if (rc != OVN_OK) return rc;
  if (!h->train && (rc = train_alloc(h)) != OVN_OK) return rc;
  const size_t bytes = (size_t)(whole_network ? h->params.n_total : h->params.n_head) * sizeof(float);
  OVN_CUDA(h, cudaMemcpyAsync(h->train->accum, d_in, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return OVN_OK;
}

int ovn_adagrad_step_sum(ovn_handle* h, int32_t whole_network, const float* d_parts, int32_t n_parts,
                         const float* h_weights, float learning_rate, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  if (!h->net_ok) OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_adagrad_step_sum: %s", h->net_error.c_str());
  if (h->cfg.precision != OVN_PREC_FP32)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_adagrad_step_sum: training needs a precision fp32 handle");
  if (!h->weights_ready) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "ovn_adagrad_step_sum: weights not finalised");
  REQUIRE(h, n_parts >= 1, "n_parts must be at least 1");
  if (n_parts > kMaxSumParts)
    OVN_SET_ERR(h, OVN_ERR_CAPACITY, "ovn_adagrad_step_sum: n_parts=%d exceeds %d", n_parts, kMaxSumParts);
  REQUIRE(h, d_parts && h_weights, "NULL pointer");
  REQUIRE(h, !h->train || h->train->stage_np == 0 || h->train->stage_stop == -1,
          "the last gradient call stopped at a stage (ovn_set_train_stop): its parts are not gradients");
  if (!h->train) {
    int rc = train_alloc(h);
    if (rc != OVN_OK) return rc;
  }
  return adagrad_sum_fp32(h, whole_network != 0, d_parts, n_parts, h_weights, learning_rate, (cudaStream_t)stream);
}

int ovn_gather_images(ovn_handle* h, const float* d_images, int64_t n_images, const int32_t* d_rows,
                      const int32_t* d_shift, const float* d_rot, int32_t n, float* d_out, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n > 0 && n_images > 0, "n and n_images must be positive");
  REQUIRE(h, d_images && d_rows && d_out, "NULL pointer");
  return gather_images(h, d_images, n_images, d_rows, d_shift, d_rot, n, d_out, (cudaStream_t)stream);
}

// ---- a training image bank in host memory -------------------------------------------------------------------
int ovn_train_workspace_bytes(ovn_handle* h, int32_t whole_network, int32_t n_pairs, int64_t* bytes) {
  if (!h) return OVN_ERR_INVALID_ARG;
  REQUIRE(h, bytes, "NULL pointer");
  REQUIRE(h, n_pairs > 0, "n_pairs must be positive");
  if (!h->net_ok) OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_train_workspace_bytes: %s", h->net_error.c_str());
  *bytes = train_workspace_bytes(h, whole_network != 0, n_pairs);
  return OVN_OK;
}

int ovn_host_register(ovn_handle* h, void* h_ptr, int64_t bytes) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, h_ptr && bytes > 0, "NULL pointer or no bytes");
  OVN_CUDA(h, cudaHostRegister(h_ptr, (size_t)bytes, cudaHostRegisterPortable));
  return OVN_OK;
}

int ovn_host_unregister(ovn_handle* h, void* h_ptr) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, h_ptr, "NULL pointer");
  OVN_CUDA(h, cudaHostUnregister(h_ptr));
  return OVN_OK;
}

int ovn_stage_rows(ovn_handle* h, const void* h_src, int64_t n_src_rows, int64_t row_bytes, const int64_t* h_rows,
                   int32_t n, void* d_dst, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n >= 0 && n_src_rows >= 0 && row_bytes > 0, "negative size");
  REQUIRE(h, n == 0 || (h_src && h_rows && d_dst), "NULL pointer");
  for (int32_t i = 0; i < n; ++i)          // all rows first: a refused call copies nothing
    if (h_rows[i] < 0 || h_rows[i] >= n_src_rows)
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_stage_rows: row %lld of entry %d is outside [0, %lld)",
                  (long long)h_rows[i], i, (long long)n_src_rows);
  const char* src = (const char*)h_src;
  char* dst = (char*)d_dst;
  for (int32_t i = 0; i < n; ++i)
    OVN_CUDA(h, cudaMemcpyAsync(dst + (size_t)i * row_bytes, src + (size_t)h_rows[i] * row_bytes, (size_t)row_bytes,
                                cudaMemcpyHostToDevice, (cudaStream_t)stream));
  return OVN_OK;
}

// ---- a training image bank sharded over the GPUs of a node --------------------------------------------------
static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ovn_shard_create writes 64 bytes of IPC handle");

int ovn_shard_create(ovn_handle* h, int64_t bytes, void** d_ptr, void* h_ipc) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, d_ptr && h_ipc, "NULL pointer");
  REQUIRE(h, bytes > 0, "bytes must be positive");
  *d_ptr = nullptr;
  Buffer<uint8_t> shard;
  int rc = shard.ensure(h, (size_t)bytes);          // exactly `bytes`: the IPC handle names the allocation's base
  if (rc != OVN_OK) return rc;
  cudaIpcMemHandle_t ipc;
  OVN_CUDA(h, cudaIpcGetMemHandle(&ipc, shard.get()));
  memcpy(h_ipc, &ipc, sizeof(ipc));
  *d_ptr = shard.get();
  h->own_shards.push_back(std::move(shard));
  return OVN_OK;
}

int ovn_shard_open(ovn_handle* h, const void* h_ipc, void** d_ptr) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, d_ptr && h_ipc, "NULL pointer");
  *d_ptr = nullptr;
  cudaIpcMemHandle_t ipc;
  memcpy(&ipc, h_ipc, sizeof(ipc));
  void* p = nullptr;
  OVN_CUDA(h, cudaIpcOpenMemHandle(&p, ipc, cudaIpcMemLazyEnablePeerAccess));
  h->open_shards.emplace_back(p);
  *d_ptr = p;
  return OVN_OK;
}

int ovn_shard_close(ovn_handle* h, void* d_ptr) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, d_ptr, "NULL pointer");
  for (size_t i = 0; i < h->open_shards.size(); ++i)
    if (h->open_shards[i].get() == d_ptr) {
      OVN_CUDA(h, cudaDeviceSynchronize());           // no queued gather still reads the mapping
      h->open_shards.erase(h->open_shards.begin() + i);
      return OVN_OK;
    }
  for (size_t i = 0; i < h->own_shards.size(); ++i)
    if (h->own_shards[i].get() == d_ptr) {
      OVN_CUDA(h, cudaDeviceSynchronize());
      h->own_shards.erase(h->own_shards.begin() + i);
      return OVN_OK;
    }
  OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_shard_close: %p is neither a shard of this handle nor one it opened", d_ptr);
}

int ovn_gather_rows(ovn_handle* h, const void* const* h_shards, const int64_t* h_first, int32_t n_shards,
                    int64_t row_bytes, const int64_t* h_rows, int32_t n, void* d_dst, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n >= 0, "n must not be negative");
  REQUIRE(h, n_shards >= 1, "n_shards must be at least 1");
  REQUIRE(h, h_shards && h_first, "NULL shard table");
  REQUIRE(h, row_bytes > 0 && row_bytes % 16 == 0, "row_bytes must be a positive multiple of 16");
  REQUIRE(h, h_first[0] == 0, "h_first[0] must be 0");
  for (int32_t s = 0; s < n_shards; ++s) {
    if (h_first[s + 1] < h_first[s])
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_gather_rows: h_first decreases at shard %d", s);
    if (!h_shards[s] || (uintptr_t)h_shards[s] % 16 != 0)
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_gather_rows: shard %d pointer %p is NULL or not 16-byte aligned", s,
                  h_shards[s]);
  }
  if (n == 0) return OVN_OK;
  REQUIRE(h, h_rows && d_dst, "NULL pointer");
  REQUIRE(h, (uintptr_t)d_dst % 16 == 0, "d_dst is not 16-byte aligned");
  const int64_t n_rows = h_first[n_shards];
  std::vector<const void*> src(n);
  for (int32_t i = 0; i < n; ++i) {                    // all rows first: a refused call copies nothing
    const int64_t r = h_rows[i];
    if (r < 0 || r >= n_rows)
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_gather_rows: row %lld of entry %d is outside [0, %lld)", (long long)r, i,
                  (long long)n_rows);
    // the last shard whose first row is <= r: an empty shard before it has the same first row
    const int32_t s = (int32_t)(std::upper_bound(h_first, h_first + n_shards + 1, r) - h_first) - 1;
    src[i] = static_cast<const uint8_t*>(h_shards[s]) + (r - h_first[s]) * row_bytes;
  }
  return gather_rows(h, src.data(), n, row_bytes, d_dst, (cudaStream_t)stream);
}

int ovn_bank_prepare(ovn_handle* h, const float* d_bank, int64_t bank_capacity, int64_t first, int64_t count,
                     void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, d_bank != nullptr, "d_bank is NULL");
  REQUIRE(h, bank_capacity > 0 && first >= 0 && count >= 0 && first + count <= bank_capacity, "bad row range");
  if (h->cfg.precision != OVN_PREC_F16_TC || count == 0) return OVN_OK;
  if (!h->weights_ready) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "ovn_bank_prepare: weights not finalised");
  int rc = tc_bank_prepare(h, d_bank, bank_capacity, first, count, (cudaStream_t)stream);
  if (rc == OVN_OK) OVN_CUDA(h, cudaEventRecord(h->ev_bank, (cudaStream_t)stream));
  return rc;
}

int ovn_peer_signal(ovn_handle* h, const uint64_t* h_flag_ptrs, int32_t n, int32_t value, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  if (n == 0) return OVN_OK;
  REQUIRE(h, h_flag_ptrs != nullptr && n > 0 && n <= 16, "bad peer list (at most 16 peers)");
  PeerPtrs pp = {};
  for (int i = 0; i < n; ++i) pp.p[i] = reinterpret_cast<int32_t*>(h_flag_ptrs[i]);
  k_peer_signal<<<1, 32, 0, (cudaStream_t)stream>>>(pp, n, value);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

int ovn_peer_wait(ovn_handle* h, const int32_t* d_flags, int32_t n, int32_t skip, int32_t value, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  if (n == 0) return OVN_OK;
  REQUIRE(h, d_flags != nullptr && n > 0 && n <= 32, "bad flag list");
  k_peer_wait<<<1, 32, 0, (cudaStream_t)stream>>>(d_flags, n, skip, value, h->d_err);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

int ovn_check(ovn_handle* h, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  return check_device_error(h, (cudaStream_t)stream);
}

int ovn_set_feature_center(ovn_handle* h, const float* h_mu) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  if (h->cfg.precision != OVN_PREC_F16_TC) return OVN_OK;
  if (!h->weights_ready) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "ovn_set_feature_center: weights not finalised");
  return tc_set_center(h, h_mu);
}

int ovn_calibrate(ovn_handle* h, const float* d_volume, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, d_volume != nullptr, "d_volume is NULL");
  if (h->cfg.precision != OVN_PREC_F16_TC) return OVN_OK;
  if (!h->weights_ready) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "ovn_calibrate: weights not finalised");
  return tc_calibrate(h, d_volume, (cudaStream_t)stream);
}

int ovn_heads_stage_pairs(ovn_handle* h, int64_t* n_pairs) {
  if (!h) return OVN_ERR_INVALID_ARG;
  REQUIRE(h, n_pairs != nullptr, "NULL pointer");
  if (h->cfg.precision != OVN_PREC_F16_TC)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_heads_stage_pairs: the stages exist on precision f16_tc handles only");
  *n_pairs = tc_heads_stage_pairs(h);
  return OVN_OK;
}

int ovn_copy_heads_stage(ovn_handle* h, int32_t stage, int64_t first, int64_t count, float* d_out, void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  if (h->cfg.precision != OVN_PREC_F16_TC)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_copy_heads_stage: the stages exist on precision f16_tc handles only");
  REQUIRE(h, stage >= OVN_STAGE_O1 && stage <= OVN_STAGE_CENTRES, "unknown ovn_heads_stage");
  return tc_copy_heads_stage(h, stage, first, count, d_out, (cudaStream_t)stream);
}

int ovn_leg_stage(ovn_handle* h, const float* d_input, int32_t n_scans, int32_t layer, float* d_hi, float* d_lo,
                  void* stream) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  if (h->cfg.precision != OVN_PREC_F16_TC)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_leg_stage: the hi / lo planes exist on precision f16_tc handles only");
  if (!h->net_ok) OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_leg_stage: %s", h->net_error.c_str());
  if (!h->weights_ready) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "ovn_leg_stage: weights not finalised");
  REQUIRE(h, d_input && d_hi && d_lo, "NULL pointer");
  REQUIRE(h, n_scans >= 1 && n_scans <= h->cfg.max_batch_scans, "n_scans outside [1, max_batch_scans]");
  REQUIRE(h, layer >= 0 && layer <= h->n_leg - 2, "layer outside [0, leg layers - 2]");
  return tc_leg_stage(h, d_input, n_scans, layer, d_hi, d_lo, (cudaStream_t)stream);
}

int ovn_get_feature_center(ovn_handle* h, float* h_mu, int32_t* is_set) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, h_mu && is_set, "NULL pointer");
  if (h->cfg.precision != OVN_PREC_F16_TC || !h->weights_ready) {
    for (int c = 0; c < kFeatC; ++c) h_mu[c] = 0.f;
    *is_set = 0;
    return OVN_OK;
  }
  return tc_get_center(h, h_mu, is_set);
}

int ovn_bank_release(ovn_handle* h, const float* d_bank) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  if (h->cfg.precision != OVN_PREC_F16_TC) return OVN_OK;
  return tc_bank_release(h, d_bank);
}

// ---- host-buffer entry points ---------------------------------------------------------------------
// d_stage_points holds the staged cloud, [n_points][4], then its probabilities, [n_points][n_prob]
static int ensure_stage(ovn_handle* h, int64_t n_points, int n_prob = 0) {
  const size_t point_bytes = (4 + n_prob) * sizeof(float);
  const int rc = h->d_stage_points.ensure(h, n_points * point_bytes, (n_points + n_points / 8 + 4096) * point_bytes);
  if (rc != OVN_OK) return rc;
  return h->d_stage_offsets.ensure(h, ((size_t)h->cfg.max_batch_scans + 1) * sizeof(int64_t));
}

// ovn_encode_clouds_host and ovn_encode_clouds_probs_host after their argument checks; h_probs is NULL or
// [n_points][n_prob_channels]
static int encode_clouds_host(ovn_handle* h, const float* h_points, const int64_t* h_offsets, int32_t n_scans,
                              const float* h_probs, float* h_fv) {
  cudaStream_t s = h->own_stream;
  const int Wf = h->cfg.leg_output_width;
  const int n_prob = h_probs ? h->cfg.n_prob_channels : 0;
  Buffer<float> d_fv;
  int rc = d_fv.ensure(h, (size_t)h->cfg.max_batch_scans * Wf * kFeatC * sizeof(float));
  if (rc != OVN_OK) return rc;
  for (int s0 = 0; s0 < n_scans; s0 += h->cfg.max_batch_scans) {
    const int n = (n_scans - s0 < h->cfg.max_batch_scans) ? n_scans - s0 : h->cfg.max_batch_scans;
    const int64_t p0 = h_offsets[s0], p1 = h_offsets[s0 + n];
    rc = ensure_stage(h, p1 - p0, n_prob);
    if (rc != OVN_OK) return rc;
    std::vector<int64_t> rel(n + 1);
    for (int i = 0; i <= n; ++i) rel[i] = h_offsets[s0 + i] - p0;
    OVN_CUDA(h, cudaMemcpyAsync(h->d_stage_points, h_points + p0 * 4, (p1 - p0) * 4 * sizeof(float),
                                cudaMemcpyHostToDevice, s));
    float* d_probs = nullptr;
    if (n_prob > 0) {
      d_probs = h->d_stage_points + (p1 - p0) * 4;
      OVN_CUDA(h, cudaMemcpyAsync(d_probs, h_probs + p0 * n_prob, (p1 - p0) * n_prob * sizeof(float),
                                  cudaMemcpyHostToDevice, s));
    }
    OVN_CUDA(h, cudaMemcpyAsync(h->d_stage_offsets, rel.data(), (n + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    OVN_CUDA(h, cudaStreamSynchronize(s));   // rel is a stack-lifetime buffer
    rc = preprocess_cues_batch(h, h->d_stage_points, h->d_stage_offsets, n, p1 - p0, d_probs, h->d_input, s);
    if (rc == OVN_OK) rc = ovn_leg_forward(h, h->d_input, n, d_fv, s);
    if (rc != OVN_OK) return rc;
    OVN_CUDA(h, cudaMemcpyAsync(h_fv + (size_t)s0 * Wf * kFeatC, d_fv, (size_t)n * Wf * kFeatC * sizeof(float),
                                cudaMemcpyDeviceToHost, s));
    rc = check_device_error(h, s);           // synchronises s
    if (rc != OVN_OK) return rc;
  }
  return OVN_OK;
}

int ovn_encode_clouds_host(ovn_handle* h, const float* h_points, const int64_t* h_offsets, int32_t n_scans,
                           float* h_fv) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_scans >= 0, "negative size");
  if (n_scans == 0) return OVN_OK;
  REQUIRE(h, h_points && h_offsets && h_fv, "NULL pointer");
  if (h->cfg.n_prob_channels != 0)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_encode_clouds_host: semantic channels need per-point probabilities; "
                "use the device-pointer stages");
  return encode_clouds_host(h, h_points, h_offsets, n_scans, nullptr, h_fv);
}

int ovn_encode_clouds_probs_host(ovn_handle* h, const float* h_points, const int64_t* h_offsets, int32_t n_scans,
                                 const float* h_probs, float* h_fv) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_scans >= 0, "negative size");
  if (n_scans == 0) return OVN_OK;
  REQUIRE(h, h_points && h_offsets && h_fv, "NULL pointer");
  REQUIRE(h, (h_probs != nullptr) == (h->cfg.n_prob_channels != 0),
          "h_probs must be given exactly when the handle has probability channels");
  return encode_clouds_host(h, h_points, h_offsets, n_scans, h_probs, h_fv);
}

// ovn_query_cloud_vs_bank_host and ovn_query_cloud_probs_vs_bank_host after their argument checks
static int query_cloud_vs_bank_host(ovn_handle* h, const float* h_points, int64_t n_points, const float* h_probs,
                                    const float* d_bank, int64_t bank_size, const int32_t* h_cand_idx,
                                    int32_t n_cand, float* h_overlap, int32_t* h_yaw, float* h_query_fv) {
  if (n_cand > h->cfg.max_batch_pairs)
    OVN_SET_ERR(h, OVN_ERR_CAPACITY, "n_cand=%d exceeds max_batch_pairs=%d", n_cand, h->cfg.max_batch_pairs);
  cudaStream_t s = h->own_stream;
  const int n_prob = h_probs ? h->cfg.n_prob_channels : 0;
  int rc = ensure_stage(h, n_points, n_prob);
  if (rc != OVN_OK) return rc;
  const int Wf = h->cfg.leg_output_width;
  // Everything the device reads or writes asynchronously lives in the pinned staging, so the call has ONE host sync.
  int64_t* p_offs = h->stage()->offsets;
  int32_t* p_idx = h->stage_cand_idx();
  float* p_ov = h->stage_overlap();
  int32_t* p_yaw = h->stage_yaw();
  p_offs[0] = 0; p_offs[1] = n_points;
  // the bank's operand copies may have been prepared on another stream (ovn_bank_prepare records ev_bank)
  OVN_CUDA(h, cudaStreamWaitEvent(s, h->ev_bank, 0));
  OVN_CUDA(h, cudaMemcpyAsync(h->d_stage_points, h_points, (size_t)n_points * 4 * sizeof(float), cudaMemcpyHostToDevice, s));
  float* d_probs = nullptr;
  if (n_prob > 0) {
    d_probs = h->d_stage_points + (size_t)n_points * 4;
    OVN_CUDA(h, cudaMemcpyAsync(d_probs, h_probs, (size_t)n_points * n_prob * sizeof(float), cudaMemcpyHostToDevice, s));
  }
  OVN_CUDA(h, cudaMemcpyAsync(h->d_stage_offsets, p_offs, 2 * sizeof(int64_t), cudaMemcpyHostToDevice, s));
  if (h_cand_idx && n_cand > 0) {
    memcpy(p_idx, h_cand_idx, (size_t)n_cand * sizeof(int32_t));
    OVN_CUDA(h, cudaMemcpyAsync(h->d_cand_idx, p_idx, (size_t)n_cand * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  }
  rc = preprocess_cues_batch(h, h->d_stage_points, h->d_stage_offsets, 1, n_points, d_probs, h->d_input, s);
  if (rc != OVN_OK) return rc;
  rc = ovn_leg_forward(h, h->d_input, 1, h->d_query_fv, s);
  if (rc != OVN_OK) return rc;
  if (n_cand > 0) {
    if (!h_cand_idx) {
      k_iota<<<(n_cand + 255) / 256, 256, 0, s>>>(h->d_cand_idx, n_cand, 0);
      OVN_LAUNCH_CHECK(h);
    }
    rc = heads_dispatch(h, d_bank, bank_size, h->d_query_fv, h->d_cand_idx, nullptr, n_cand, h->d_query_overlap,
                        h->d_query_yaw, nullptr, s);
    if (rc != OVN_OK) return rc;
    OVN_CUDA(h, cudaMemcpyAsync(p_ov, h->d_query_overlap, (size_t)n_cand * sizeof(float), cudaMemcpyDeviceToHost, s));
    OVN_CUDA(h, cudaMemcpyAsync(p_yaw, h->d_query_yaw, (size_t)n_cand * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  }
  if (h_query_fv)
    OVN_CUDA(h, cudaMemcpyAsync(h_query_fv, h->d_query_fv, (size_t)Wf * kFeatC * sizeof(float), cudaMemcpyDeviceToHost, s));
  rc = check_device_error(h, s);            // the one synchronisation of the call
  if (n_cand > 0) {                         // results are delivered even on error (poisoned: NaN / INT32_MIN)
    memcpy(h_overlap, p_ov, (size_t)n_cand * sizeof(float));
    memcpy(h_yaw, p_yaw, (size_t)n_cand * sizeof(int32_t));
  }
  return rc;
}

int ovn_query_cloud_vs_bank_host(ovn_handle* h, const float* h_points, int64_t n_points, const float* d_bank,
                                 int64_t bank_size, const int32_t* h_cand_idx, int32_t n_cand, float* h_overlap,
                                 int32_t* h_yaw, float* h_query_fv) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_points >= 0 && n_cand >= 0, "negative size");
  REQUIRE(h, h_points, "h_points is NULL");
  REQUIRE(h, n_cand == 0 || (d_bank && h_overlap && h_yaw), "NULL pointer");
  REQUIRE(h, n_cand == 0 || bank_size > 0, "bank_size must be positive");
  REQUIRE(h, h_cand_idx != nullptr || n_cand <= bank_size, "n_cand exceeds bank_size");
  if (h->cfg.n_prob_channels != 0)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "ovn_query_cloud_vs_bank_host: semantic channels are not supported here");
  return query_cloud_vs_bank_host(h, h_points, n_points, nullptr, d_bank, bank_size, h_cand_idx, n_cand, h_overlap,
                                  h_yaw, h_query_fv);
}

int ovn_query_cloud_probs_vs_bank_host(ovn_handle* h, const float* h_points, int64_t n_points, const float* h_probs,
                                       const float* d_bank, int64_t bank_size, const int32_t* h_cand_idx,
                                       int32_t n_cand, float* h_overlap, int32_t* h_yaw, float* h_query_fv) {
  if (!h) return OVN_ERR_INVALID_ARG;
  DeviceGuard guard(h);
  REQUIRE(h, n_points >= 0 && n_cand >= 0, "negative size");
  REQUIRE(h, h_points, "h_points is NULL");
  REQUIRE(h, n_cand == 0 || (d_bank && h_overlap && h_yaw), "NULL pointer");
  REQUIRE(h, n_cand == 0 || bank_size > 0, "bank_size must be positive");
  REQUIRE(h, h_cand_idx != nullptr || n_cand <= bank_size, "n_cand exceeds bank_size");
  REQUIRE(h, (h_probs != nullptr) == (h->cfg.n_prob_channels != 0),
          "h_probs must be given exactly when the handle has probability channels");
  return query_cloud_vs_bank_host(h, h_points, n_points, h_probs, d_bank, bank_size, h_cand_idx, n_cand, h_overlap,
                                  h_yaw, h_query_fv);
}

}  // extern "C"
