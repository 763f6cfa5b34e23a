// Engine internals: network description, packed weights, workspace arena.
#pragma once
#include <cufft.h>

#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/sgmse_b200.h"
#include "kernels.h"

namespace sgmse {

struct ParamRef {       // one state_dict() entry
  std::string name;
  long long numel = 0;
  long long offset = 0; // floats from the start of the blob
};

struct ConvW {          // packed convolution weights (K ordering: segment, tap, cin)
  void* w_direct = nullptr;   // [Ktot][Cout] float or half
  __half* w_tc = nullptr;     // [Cout][w_tc_ld], K-major; optional identity tail (see pack_conv)
  int w_tc_ld = 0;
  bool identity_tail = false;
  float* bias = nullptr;      // [Cout] fp32 (device)
  int ktot = 0, cout = 0;
};

enum LayerKind { LK_RES, LK_ATTN, LK_COMBINE, LK_OUTCONV /* GN + conv3x3(C->4) pair */ };

struct Layer {
  LayerKind kind;
  int idx = 0;          // index into all_modules (first module of the pair for LK_OUTCONV)
  int cin = 0, cout = 0;
  bool up = false, down = false, shortcut = false;
  int temb_off = 0;     // column offset into the temb table (LK_RES)
  // parameter offsets into the fp32 blob
  long long gn0_w = -1, gn0_b = -1, gn1_w = -1, gn1_b = -1;
  long long conv0_w = -1, conv0_b = -1, conv1_w = -1, conv1_b = -1, conv2_w = -1, conv2_b = -1;
  long long dense_w = -1, dense_b = -1;
  long long nin_w[4] = {-1, -1, -1, -1}, nin_b[4] = {-1, -1, -1, -1};
  // packed
  ConvW c0, c1;         // LK_RES: Conv_0, Conv_1(+Conv_2); LK_ATTN: qkv, proj
  float* small_w = nullptr;   // LK_COMBINE: [4][C]; LK_OUTCONV: [9C][4]
  float* small_b = nullptr;   // LK_COMBINE: [C] (device)
  float out_bias_host[4] = {0, 0, 0, 0};
  uint2* small_wfrag = nullptr;   // LK_OUTCONV: mma.sync B fragments [9][C/16][32] of small_w in fp16 (see out_conv_mma_kernel)
};

struct Arena {
  uint8_t* base = nullptr;
  size_t cap = 0, off = 0, high = 0;
  bool dry = false;
  void* alloc(size_t bytes) {
    off = (off + 255) & ~(size_t)255;
    void* p = base ? base + off : reinterpret_cast<void*>(off);
    off += bytes;
    if (off > high) high = off;
    if (!dry) SG_CHECK(off <= cap, "workspace overflow: need %zu, have %zu", off, cap);
    return p;
  }
  void reset() { off = 0; }
};

struct GraphKey {
  int B, F, T, N, pred, corr, csteps, denoise, pf;
  float snr;
  int kind;
  float sb_eps;
  bool operator<(const GraphKey& o) const {
    return std::tie(B, F, T, N, pred, corr, csteps, denoise, pf, snr, kind, sb_eps) <
           std::tie(o.B, o.F, o.T, o.N, o.pred, o.corr, o.csteps, o.denoise, o.pf, o.snr, o.kind, o.sb_eps);
  }
};

struct ConvTiming {
  cudaEvent_t start, stop;
  double flops, bytes;
  bool tc;
};

struct GraphEntry {
  cudaGraphExec_t exec;
  long long kernel_nodes;
  long long last_used = 0;   // engine.graph_clock at the last launch (least-recently-used eviction)
};

struct FwdGraph {            // one captured score-network evaluation on e.state (ODE sampler: t changes per evaluation)
  cudaGraphExec_t exec;
  const float4* out;         // the network's 4-channel output pyramid (arena address, stable per shape)
  long long kernel_nodes;
  long long tc_convs, direct_convs;
};

struct OdeBuffers {          // state of the probability-flow ODE sampler for one whole batch (SURVEY.md §8f-4)
  double2* y = nullptr;      // complex128 like scipy's integrator state
  double2* y_new = nullptr;
  float2* k[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // complex64 stage derivatives
  float2* stage = nullptr;   // complex64 argument of the next evaluation
  double* partial = nullptr; // [kOdeNormBlocks] device
  double* partial_host = nullptr;   // pinned
  size_t cap_px = 0;
};

}  // namespace sgmse

struct sgmse_b200_engine {
  sgmse_b200_config cfg{};
  std::vector<sgmse::ParamRef> manifest;
  long long weights_numel = 0;
  std::vector<sgmse::Layer> layers;           // execution order (= all_modules order of block-level modules)
  int total_temb_c = 0;
  // blob offsets of the non-block parameters
  long long gfp_w = -1, lin1_w = -1, lin1_b = -1, lin2_w = -1, lin2_b = -1, inconv_w = -1, inconv_b = -1;
  long long outl_w = -1, outl_b = -1;

  // device state
  bool loaded = false;
  float* blob_dev = nullptr;                  // raw fp32 parameters (GN affine, biases, Linear weights ...)
  std::vector<void*> dev_allocs;              // packed weights etc.
  float* inconv_w_packed = nullptr;           // [36][nf]
  float* dense_w_stacked = nullptr;           // [totalC][4nf]
  float* dense_b_stacked = nullptr;           // [totalC]
  sgmse::OutLayer out_layer{};
  size_t weights_bytes = 0;

  sgmse::Arena arena;                         // activations of one forward pass
  // persistent sampler buffers (sized for max_batch)
  float4* state = nullptr;
  float2* xmean = nullptr;
  float* temb_table = nullptr;                // [rows][totalC]
  float* temb_scratch = nullptr;
  float* t_dev = nullptr;
  sgmse::UpdateCoef* coef_dev = nullptr;
  sgmse::RngParams* rng_dev = nullptr;
  float* lv_scratch = nullptr;
  int* dbg_flag = nullptr;
  unsigned int* range_flag = nullptr;         // device word, shared with the lanes: fp16 overflow events seen by GroupNorm (gn.cu)
  size_t persist_px = 0;                      // capacity of state/xmean in pixels
  int persist_rows = 0;                       // capacity of temb_table in rows

  std::map<sgmse::GraphKey, sgmse::GraphEntry> graphs;
  long long graph_clock = 0;
  int max_graphs = 16;                        // a long-running service sees many (B, T, sampler) keys: keep the 16 most recent
  std::map<std::tuple<int, int, int>, sgmse::FwdGraph> fwd_graphs;   // (B, F, T) -> captured single evaluation
  sgmse::OdeBuffers ode;
  std::map<std::tuple<int, int, int>, size_t> arena_need;   // workspace bytes per (B, F, T)
  cudaStream_t own_stream = nullptr;
  std::map<std::pair<int, int>, cufftHandle> fft_plans;   // (type<<28 | n_fft, batch)
  void* stft_buf[4] = {nullptr, nullptr, nullptr, nullptr};
  size_t stft_cap[4] = {0, 0, 0, 0};

  // Concurrent lanes: inside a captured sampler graph the micro-batch is split over `num_lanes` independent
  // launch sequences on forked streams, so that the HBM-bound kernels of one lane (GroupNorm apply, FIR, PC
  // update) overlap the tensor-bound convolutions of the other.  A lane is a shadow engine: it shares the
  // packed weights (owns_weights == false) and owns its workspace, state and staging buffers.
  int num_lanes = 1;                          // concurrent launch sequences inside a captured sampler graph (option "lanes")
  bool owns_weights = true;
  std::vector<sgmse_b200_engine*> lanes;      // lanes[0] == this
  std::vector<cudaStream_t> lane_streams;     // lane_streams[0] unused (lane 0 runs on the caller's stream)
  std::vector<cudaEvent_t> lane_events;       // [0] fork, [i] join of lane i
  long long generation = 0;                   // bumped whenever a graph-visible buffer is re-allocated
  long long lanes_generation_seen = -1;

  // Kernel A/B selection of THIS engine.  The launch helpers read thread-local switches (kernels.h: g_*); every C-ABI entry
  // point installs the calling engine's set first (engine.cu: activate), so two engines of one process -- or of two host
  // threads -- never see each other's choices, and a captured graph keeps the choices of the engine that captured it.
  struct KernelOpts {
    int tc_variant = 0, tc1_narrow = 0;
    int attn_variant = 0, fir_variant = 0, inconv_variant = 0, outconv_variant = 0, combine_variant = 0;
    int gn_self = 0, gnfin_variant = 0, pdl = 0;
  } opts;

  // options / counters
  bool record_taps = false;
  bool time_convs = false;
  std::vector<sgmse::ConvTiming> conv_events;
  long long tc_mask = -1;
  std::map<std::string, sgmse::TensorDesc> taps;
  std::map<std::string, std::pair<const float4*, std::vector<int>>> taps4;
  long long kernel_launches = 0, graph_launches = 0;
  long long tc_convs = 0, direct_convs = 0;
  long long launches_this_forward = 0;
};
