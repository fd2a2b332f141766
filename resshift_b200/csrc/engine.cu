// Engine: the Swin-UNet denoiser of ResShift as a static program of sm_90a kernel launches, plus the
// residual-shift, DDPM / DDIM and DDIM-inversion sampling loops, behind the C ABI declared in include/resshift_b200.h.
//
// Topology restates UNetModelSwin.__init__/forward (reference models/unet.py:659-895), ResBlock
// (:110-206), BasicLayer / SwinTransformerBlock (models/swin_transformer.py:163-281,348-442).
// Design notes (DESIGN.md has the long form):
//   * activations NHWC fp16; skip connections are written straight into the channel slice of the
//     decoder's concat buffer (th.cat at unet.py:891 costs nothing);
//   * every tensor lives in one caller-owned workspace; lifetimes are resolved at plan time;
//   * timestep embeddings (time_embed + all 22 emb_layers) are one small table computed by two tiny
//     kernels; in the sampling loop the table for all T steps is computed once.
#include <algorithm>
#include <cmath>
#include <map>
#include <memory>
#include <numeric>
#include <optional>
#include <string>
#include <variant>
#include <vector>

#include "../../include/resshift_b200.h"
#include "launch.cuh"
#include "vq_kernels.cuh"

namespace rs {

static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
int fail(int code, const std::string& msg) { g_last_error = msg; return code; }

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

enum Role { R_CONV3 = 0, R_CONV1, R_LINEAR, R_BIAS, R_GN_W, R_GN_B, R_RELPOS, R_BUF_RELIDX, R_BUF_MASK, R_F32 /* fp32 tensor kept as is (VQ codebook) */ };

struct Param {
  std::string name;
  std::vector<int> shape;
  int role;
  size_t off = 0;        // byte offset in the arena
  size_t bytes = 0;
  int ipad = 0;          // padded input channels for weights
};

}  // namespace rs

using namespace rs;

namespace {
enum class EngineKind { Denoiser, VqGan, Kl };   // the denoiser or a first stage around it (vq.inc)
enum class Pass { Denoiser, Encode, Decode };    // a plan's program: the denoiser's forward, a first stage's encoder / decoder
const char* kind_name(EngineKind k) {
  switch (k) {
    case EngineKind::Denoiser: return "a UNetModelSwin denoiser";
    case EngineKind::VqGan: return "a VQ-GAN first stage";
    case EngineKind::Kl: return "a KL first stage";
  }
  return "an engine of unknown kind";
}
// launches a bound plan makes outside its op list: the denoiser's timestep embedding (4) and input packing (1-2); a first
// stage's counter reset, input packing or quantiser, and output copy
constexpr int kDenoiserOuterLaunches = 6, kEncodeOuterLaunches = 3, kDecodeOuterLaunches = 3;
}  // namespace

struct rs_engine {
  EngineKind kind = EngineKind::Denoiser;   // the parameter store is shared by all kinds
  rs_vq_config vq{};
  rs_vq_options vqopt{};                    // first stages: attention levels, mid attention, resampling, tanh (rs_vq_create_ex)
  rs_unet_config cfg;
  rs_unet_options opt{1, 0, 1, 0};
  // UNetModel (rs_unetmodel_create): global-attention blocks instead of Swin layers, no feature extractor; cfg then holds
  // its levels with in_channels = the channels of x (out_channels, or half of it with a learned variance) and
  // lq_size = image_size
  bool unetmodel = false;
  rs_unetmodel_config um{};
  // UNetModelConv (rs_unetconv_create): a UNetModel-style engine (unetmodel set, no attention levels) whose ResBlocks are
  // ResBlockConv — SiLU and conv without GroupNorm — and whose head is conv3x3(SiLU(h))
  bool conv_blocks = false;
  std::vector<Param> params;
  std::map<std::string, int> index;
  size_t arena_bytes = 0;
  uint8_t* arena = nullptr;
  int device = -1;              // CUDA device that was current at rs_unet_set_arena (where the arena lives)
  unsigned long long weights_epoch = 0;    // bumped by every rs_unet_load_param: tables derived from weights (FiLM) go stale
  // concatenated emb_layers ("FiLM") matrix: rows = sum 2*Cout over ResBlocks, K = time_embed_dim
  size_t film_w_off = 0, film_b_off = 0;
  int film_rows = 0;
  std::map<std::string, int> film_row_of;   // resblock prefix -> first row

  int time_dim() const { return cfg.model_channels * 4; }
  int fe_stages() const {
    if (cfg.lq_size == cfg.image_size) return 0;
    int s = 0, r = cfg.lq_size / cfg.image_size;
    while (r > 1) { r >>= 1; ++s; }
    return s;
  }
  int lq_in_ch() const { return cfg.cond_mask ? 4 : 3; }
  int lq_feat_ch() const {
    if (unetmodel) return um.in_channels - cfg.in_channels;     // cfg.in_channels: the channels of x
    return fe_stages() == 0 ? lq_in_ch() : 16 << fe_stages();
  }
  // UNetModel: the LQ image enters at the latent size (1) or at twice it through pixel_unshuffle (2)
  int lq_factor() const { return unetmodel && lq_feat_ch() == 4 * lq_in_ch() ? 2 : 1; }
  // heads of a UNetModel AttentionBlock over ch channels; output blocks are built without num_heads (unet.py:517-523)
  int attn_heads(int ch, bool output_block) const {
    if (um.num_head_channels != -1) return ch / um.num_head_channels;
    return output_block ? 1 : um.num_heads;
  }
  bool has_attn(int ds) const {
    for (int i = 0; i < cfg.n_attn; ++i) if (cfg.attention_resolutions[i] == ds) return true;
    return false;
  }
  const Param* find(const std::string& n) const {
    auto it = index.find(n);
    return it == index.end() ? nullptr : &params[it->second];
  }
  template <typename T> T* at(const std::string& n) const {
    const Param* p = find(n);
    return p ? reinterpret_cast<T*>(arena + p->off) : nullptr;
  }
  const __half* packed(const std::string& n, int* ld) const {   // a packed fp16 weight matrix and its row length
    const Param* p = find(n);
    if (p) *ld = p->ipad;
    return at<__half>(n);
  }
};

// ------------------------------------------------------------------------------------------------
// architecture walk shared by the parameter inventory and the plan builder
// ------------------------------------------------------------------------------------------------
namespace {

// kind: 0 conv(cin,cout) 1 res(cin,cout) 2 swin(c,res) 3 down(c) 4 up(c) 5 res with down=True(c) 6 res with up=True(c)
// 7 UNetModel AttentionBlock(c,heads)
struct Layer { int kind; int a, b; };
enum { L_CONV = 0, L_RES, L_SWIN, L_DOWN, L_UP, L_RES_DOWN, L_RES_UP, L_ATTN };
struct Topology {
  std::vector<std::vector<Layer>> input_blocks, output_blocks;
  std::vector<Layer> middle;
  std::vector<int> in_block_ch;    // output channels of each input block (the skip stack)
};

Topology build_topology(const rs_engine& e) {
  const rs_unet_config& c = e.cfg;
  Topology t;
  const int mc = c.model_channels;
  int ch = c.channel_mult[0] * mc;
  t.input_blocks.push_back({{0, c.in_channels + e.lq_feat_ch(), ch}});
  std::vector<int> chans{ch};
  int ds = c.image_size;
  // UNetModel (reference models/unet.py:426-541): an AttentionBlock after EVERY ResBlock of an attention level; the
  // Swin UNet puts a BasicLayer after the first one only
  auto add_attn = [&](std::vector<Layer>& layers, int jj, int chn, bool output_block) {
    if (!e.has_attn(ds)) return;
    if (e.unetmodel) layers.push_back({L_ATTN, chn, e.attn_heads(chn, output_block)});
    else if (jj == 0) layers.push_back({L_SWIN, chn, ds});
  };
  for (int level = 0; level < c.n_levels; ++level) {
    for (int jj = 0; jj < c.num_res_blocks[level]; ++jj) {
      std::vector<Layer> layers{{1, ch, c.channel_mult[level] * mc}};
      ch = c.channel_mult[level] * mc;
      add_attn(layers, jj, ch, false);
      t.input_blocks.push_back(layers);
      chans.push_back(ch);
    }
    if (level != c.n_levels - 1) {
      t.input_blocks.push_back({{e.opt.resblock_updown ? L_RES_DOWN : L_DOWN, ch, ch}});
      chans.push_back(ch);
      ds /= 2;
    }
  }
  t.in_block_ch = chans;
  if (e.conv_blocks) t.middle = {{1, ch, ch}, {1, ch, ch}};      // two ResBlockConv (reference models/unet.py:1103-1116)
  else t.middle = {{1, ch, ch}, {e.unetmodel ? L_ATTN : L_SWIN, ch, e.unetmodel ? e.attn_heads(ch, false) : ds}, {1, ch, ch}};
  for (int level = c.n_levels - 1; level >= 0; --level) {
    for (int i = 0; i <= c.num_res_blocks[level]; ++i) {
      const int ich = chans.back(); chans.pop_back();
      std::vector<Layer> layers{{1, ch + ich, mc * c.channel_mult[level]}};
      ch = mc * c.channel_mult[level];
      add_attn(layers, i, ch, true);
      if (level && i == c.num_res_blocks[level]) { layers.push_back({e.opt.resblock_updown ? L_RES_UP : L_UP, ch, ch}); ds *= 2; }
      t.output_blocks.push_back(layers);
    }
  }
  return t;
}

void add_param(rs_engine& e, const std::string& name, std::vector<int> shape, int role) {
  Param p; p.name = name; p.shape = std::move(shape); p.role = role;
  e.index[name] = (int)e.params.size();
  e.params.push_back(std::move(p));
}
void add_conv(rs_engine& e, const std::string& n, int cin, int cout, int k) {
  add_param(e, n + ".weight", {cout, cin, k, k}, k == 3 ? R_CONV3 : R_CONV1);
  add_param(e, n + ".bias", {cout}, R_BIAS);
}
void add_linear(rs_engine& e, const std::string& n, int cin, int cout) {
  add_param(e, n + ".weight", {cout, cin}, R_LINEAR);
  add_param(e, n + ".bias", {cout}, R_BIAS);
}
void add_gn(rs_engine& e, const std::string& n, int c) {
  add_param(e, n + ".weight", {c}, R_GN_W);
  add_param(e, n + ".bias", {c}, R_GN_B);
}

void add_layers(rs_engine& e, const std::string& prefix, const std::vector<Layer>& layers) {
  const rs_unet_config& c = e.cfg;
  for (size_t j = 0; j < layers.size(); ++j) {
    const Layer& L = layers[j];
    const std::string p = prefix + "." + std::to_string(j);
    if (L.kind == L_CONV) {
      add_conv(e, p, L.a, L.b, 3);
    } else if ((L.kind == L_RES || L.kind == L_RES_DOWN || L.kind == L_RES_UP) && e.conv_blocks) {
      // ResBlockConv (reference models/unet.py:914-982): in_layers = [SiLU, conv], out_layers = [SiLU, conv]
      const int cout = L.kind == L_RES ? L.b : L.a;
      add_conv(e, p + ".in_layers.1", L.a, cout, 3);
      add_linear(e, p + ".emb_layers.1", e.time_dim(), (e.opt.use_scale_shift_norm ? 2 : 1) * cout);
      add_conv(e, p + ".out_layers.1", cout, cout, 3);
      if (L.a != cout) add_conv(e, p + ".skip_connection", L.a, cout, 1);
    } else if (L.kind == L_RES || L.kind == L_RES_DOWN || L.kind == L_RES_UP) {
      const int cout = L.kind == L_RES ? L.b : L.a;
      add_gn(e, p + ".in_layers.0", L.a);
      add_conv(e, p + ".in_layers.2", L.a, cout, 3);
      add_linear(e, p + ".emb_layers.1", e.time_dim(), (e.opt.use_scale_shift_norm ? 2 : 1) * cout);
      add_gn(e, p + ".out_layers.0", cout);
      add_conv(e, p + ".out_layers.3", cout, cout, 3);
      if (L.a != cout) add_conv(e, p + ".skip_connection", L.a, cout, 1);
    } else if (L.kind == L_SWIN) {
      const int E = c.swin_embed_dim, res = L.b;
      const int win = res <= c.window_size ? res : c.window_size;
      const int shift = res <= c.window_size ? 0 : c.window_size / 2;
      const int hidden = (int)(E * c.mlp_ratio);
      add_conv(e, p + ".patch_embed.proj", L.a, E, 1);
      if (e.opt.patch_norm) add_gn(e, p + ".patch_embed.norm", E);
      add_conv(e, p + ".patch_unembed.proj", E, L.a, 1);
      if (e.opt.patch_norm) add_gn(e, p + ".patch_unembed.norm", L.a);
      for (int i = 0; i < c.swin_depth; ++i) {
        const std::string b = p + ".blocks." + std::to_string(i);
        if (i % 2 == 1 && shift > 0) {
          const int nw = (res / win) * (res / win);
          add_param(e, b + ".attn_mask", {nw, win * win, win * win}, R_BUF_MASK);
        }
        add_gn(e, b + ".norm1", E);
        add_param(e, b + ".attn.relative_position_bias_table", {(2 * win - 1) * (2 * win - 1), c.swin_heads}, R_RELPOS);
        add_param(e, b + ".attn.relative_position_index", {win * win, win * win}, R_BUF_RELIDX);
        add_linear(e, b + ".attn.qkv", E, 3 * E);
        add_linear(e, b + ".attn.proj", E, E);
        add_gn(e, b + ".norm2", E);
        add_conv(e, b + ".mlp.fc1", E, hidden, 1);
        add_conv(e, b + ".mlp.fc2", hidden, E, 1);
      }
    } else if (L.kind == L_ATTN) {
      // AttentionBlock (reference models/unet.py:230-255): qkv and proj_out are conv1d weights [O, I, 1], packed as 1x1 convs
      add_gn(e, p + ".norm", L.a);
      add_param(e, p + ".qkv.weight", {3 * L.a, L.a, 1}, R_CONV1);
      add_param(e, p + ".qkv.bias", {3 * L.a}, R_BIAS);
      add_param(e, p + ".proj_out.weight", {L.a, L.a, 1}, R_CONV1);
      add_param(e, p + ".proj_out.bias", {L.a}, R_BIAS);
    } else if (L.kind == L_DOWN) {
      if (e.opt.conv_resample) add_conv(e, p + ".op", L.a, L.a, 3);
    } else if (L.kind == L_UP) {
      if (e.opt.conv_resample) add_conv(e, p + ".conv", L.a, L.a, 3);
    }
  }
}

// window side w of a relative_position_bias_table [(2w-1)^2, heads]
int relpos_window(const Param& p) {
  int w = 1;
  while ((2 * w - 1) * (2 * w - 1) < p.shape[0]) ++w;
  return w;
}

int build_inventory(rs_engine& e) {
  const rs_unet_config& c = e.cfg;
  add_linear(e, "time_embed.0", c.model_channels, e.time_dim());
  add_linear(e, "time_embed.2", e.time_dim(), e.time_dim());
  int fc = e.lq_in_ch(), bc = 16;
  for (int st = 0; st < e.fe_stages(); ++st) {
    add_conv(e, "feature_extractor." + std::to_string(3 * st), fc, bc, 3);
    add_conv(e, "feature_extractor." + std::to_string(3 * st + 2) + ".op", bc, 2 * bc, 3);
    bc *= 2; fc = bc;
  }
  Topology t = build_topology(e);
  for (size_t i = 0; i < t.input_blocks.size(); ++i) add_layers(e, "input_blocks." + std::to_string(i), t.input_blocks[i]);
  add_layers(e, "middle_block", t.middle);
  for (size_t i = 0; i < t.output_blocks.size(); ++i) add_layers(e, "output_blocks." + std::to_string(i), t.output_blocks[i]);
  if (e.conv_blocks) {
    add_conv(e, "out.1", c.channel_mult[0] * c.model_channels, c.out_channels, 3);
  } else {
    add_gn(e, "out.0", c.channel_mult[0] * c.model_channels);
    add_conv(e, "out.2", c.channel_mult[0] * c.model_channels, c.out_channels, 3);
  }

  // arena layout.  emb_layers weights / biases first, contiguous, in ResBlock order, so that all of
  // them form ONE [film_rows, time_dim] matrix for a single small-linear launch.
  size_t off = 0;
  const int K = e.time_dim();
  e.film_w_off = off;
  int rows = 0;
  for (Param& p : e.params) {
    if (p.role == R_LINEAR && p.name.find(".emb_layers.1.weight") != std::string::npos) {
      p.ipad = K; p.off = off; p.bytes = (size_t)p.shape[0] * K * 2;
      e.film_row_of[p.name.substr(0, p.name.size() - std::string(".emb_layers.1.weight").size())] = rows;
      rows += p.shape[0];
      off += p.bytes;
    }
  }
  e.film_rows = rows;
  off = align_up(off, 256);
  e.film_b_off = off;
  // Without scale-shift norm the FiLM row of a ResBlock is emb_out, added to in_layers.2's output by that conv's epilogue
  // in place of its bias: the table's bias there is emb_layers.1.bias + in_layers.2.bias (rs_unet_load_param folds them),
  // and both parameters keep slots of their own below.
  for (Param& p : e.params) {
    if (p.role == R_BIAS && p.name.find(".emb_layers.1.bias") != std::string::npos) {
      if (e.opt.use_scale_shift_norm) { p.off = off; p.bytes = (size_t)p.shape[0] * 4; }
      off += (size_t)p.shape[0] * 4;
    }
  }
  off = align_up(off, 256);
  for (Param& p : e.params) {
    if (p.bytes) continue;
    switch (p.role) {
      case R_CONV3: case R_CONV1:
        p.ipad = (p.shape[1] + 7) / 8 * 8;
        p.bytes = (size_t)p.shape[0] * (p.shape.size() == 4 ? p.shape[2] * p.shape[3] : 1) * p.ipad * 2; break;   // (conv1d [O, I, 1])
      case R_LINEAR:
        p.ipad = (p.shape[1] + 7) / 8 * 8;
        p.bytes = (size_t)p.shape[0] * p.ipad * 2; break;
      case R_BIAS: case R_GN_W: case R_GN_B:
        p.bytes = (size_t)p.shape[0] * 4; break;
      case R_RELPOS: {    // expanded at load time to dense [heads][w*w][w*w] fp32
        const int w = relpos_window(p);
        p.bytes = (size_t)c.swin_heads * w * w * w * w * 4; break;
      }
      default: p.bytes = 0; break;     // buffers are derived, not stored
    }
    if (p.bytes) { p.off = off; off = align_up(off + p.bytes, 256); }
  }
  e.arena_bytes = align_up(off, 256);
  return 0;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// plan
// ------------------------------------------------------------------------------------------------
namespace {

struct Tensor {
  size_t bytes = 0;
  int first = 1 << 30, last = -1;
  size_t off = 0;
  bool persistent = false;
};

// The GroupNorm statistics a consumer reads (a GroupNorm op, the fused Swin attention's norm1):
// (mean, M2) pairs [N][slots][C][2] of `in` from its producers' epilogues (fused) or from gn_stats_kernel
struct GnLink {
  View in;
  bool fused = false;
  int slots = 0;           // pair slots per image: 128-pixel conv tiles, 8x8 windows (win_slots), or gn_chunks (unfused)
  bool win_slots = false;  // the producer is the fused Swin attention kernel: one slot per 8x8 window (64 values each)
  size_t stats_off = 0;    // offset of the pair buffer inside the stats region
  int gn_index = -1;       // index of its [N][32][2] group statistics / [N] arrival counters
  float eps = 1e-5f;
};
struct StatDst { GnLink to; int coff; };            // a consumer a producer's epilogue delivers to, at its channel coff
struct Producer { std::vector<StatDst> stat_dst; };   // conv, fused MLP, fused Swin attention: up to two consumers

// The payload of each op kind; parameter names are resolved at bind
struct ConvOp : Producer {
  ConvDesc d;
  std::string w_name, b_name;   // (b_name empty: no bias)
  int bias_film_off = -1;       // the bias is a FiLM-table row (ResBlock without scale-shift norm): its offset in a row
  int film_off = -1;            // FiLM after the activation (ResBlockConv with scale-shift norm): its [2 Cout] slice of a row
  bool to_f32 = false;          // writes the fp32 NCHW model output
  int split_tens = -1;          // workspace tensor holding split-K partial sums (or -1)
  // VQ-GAN attention GEMMs (vq.inc): "weights" that are an activation tensor [Cout rows][K] of the plan, and / or input
  // "pixels" that are the rows of the arena's weight matrix in_param (the transposed value projection)
  View w_view; bool w_is_view = false;
  std::string in_param;
};
struct GnOp { GnDesc d; GnLink stats; std::string name; };   // d.in / fused / slots / eps come from stats at bind
struct WinAttnOp {   // (simt: the SIMT cross-check kernel instead of a window_attn_kernel instance)
  View qkv, out; int window = 8, shift = 0; bool simt = false; std::string bias_name; const float* bias = nullptr;
};
struct ResampleOp { View in, out; bool pool = false; View silu; bool has_silu = false; };   // 2x nearest upsample, or (pool) 2x2
                                                                                            // average pool (+ SiLU twin of out)
struct MlpOp : Producer { MlpDesc d; std::string name; };
struct SwinOp : Producer { SwinAttnDesc d; std::string blk; GnLink norm1; };
struct SoftmaxOp { View view; float scale = 1.f; };         // in place on view [rows = N*H*W][cols = C]

// an op is its kind's payload and nothing else: the alternatives follow OpKind
enum OpKind { OP_CONV, OP_GN, OP_ATTN, OP_UPSAMPLE, OP_MLP, OP_SOFTMAX, OP_SWIN_ATTN, OP_VQ_ATTN, OP_UNET_ATTN };
using OpPayload = std::variant<ConvOp, GnOp, WinAttnOp, ResampleOp, MlpOp, SoftmaxOp, SwinOp, VqAttnDesc, UnetAttnDesc>;
template <OpKind K, typename T> constexpr bool payload_of = std::is_same_v<std::variant_alternative_t<K, OpPayload>, T>;
static_assert(std::variant_size_v<OpPayload> == OP_UNET_ATTN + 1 && payload_of<OP_CONV, ConvOp> && payload_of<OP_GN, GnOp> &&
              payload_of<OP_ATTN, WinAttnOp> && payload_of<OP_UPSAMPLE, ResampleOp> && payload_of<OP_MLP, MlpOp> &&
              payload_of<OP_SOFTMAX, SoftmaxOp> && payload_of<OP_SWIN_ATTN, SwinOp> && payload_of<OP_VQ_ATTN, VqAttnDesc> &&
              payload_of<OP_UNET_ATTN, UnetAttnDesc>);
using Op = OpPayload;
inline OpKind kind_of(const Op& op) { return static_cast<OpKind>(op.index()); }
// the payload of an op of kind T (read under that kind's case only)
template <typename T, typename O> auto& payload(O& op) { return *std::get_if<T>(&op); }

inline SoftmaxParams softmax_params(const SoftmaxOp& s) {
  const View& v = s.view;
  return SoftmaxParams{v.ptr, (long long)v.ld, v.N * v.H * v.W, v.C, s.scale};
}

}  // namespace

struct rs_plan {
  rs_engine* e = nullptr;
  Overrides ovr;             // the environment's kernel-choice overrides when the plan was created: its every decision follows them
  int B = 0, H = 0, W = 0, lqH = 0, lqW = 0;
  std::vector<Tensor> tensors;
  std::vector<Op> fe_ops, ops;
  std::map<std::string, View> block_out;
  // fixed regions (byte offsets in the workspace)
  size_t off_emb_sin = 0, off_emb_mid = 0, off_emb_vec = 0, off_film = 0, off_tsteps = 0, off_tables = 0;
  size_t off_stats = 0, stats_bytes = 0, off_state = 0, off_temps = 0, temps_bytes = 0;
  size_t off_gstat = 0, off_counters = 0;   // per GroupNorm: [N][32][2] floats (mean, rstd); [N] arrival counters
  int n_gn = 0;
  size_t workspace_bytes = 0;
  int max_rows = 0;          // rows of the FiLM table (max(B, 64) so a sampler with T <= 64 fits)
  uint8_t* ws = nullptr;
  View xin, lq_feat, fe_in;  // packed denoiser input, LQ feature (if a feature extractor exists), its input
  int cin_pad = 0, fe_cpad = 0;
  float* out_f32 = nullptr;  // model output (fp32 NCHW), inside the state region
  bool bound = false;
  int device = -1;           // CUDA device that was current at rs_plan_bind: the only one the plan runs on
  int launches = 0;
  Pass pass = Pass::Denoiser;
  int imgH = 0, imgW = 0;    // VQ plans: image size (H, W above are the latent size)
  std::vector<int> vq_attn_ops;  // VQ plans: indices in ops of the fused attentions (T > 8192), in pass order
  int vq_next = 0;           // VQ plans: the fused attention whose segment runs next (1 after _begin; 0 after _end)
  // The schedule tables and the FiLM table live in this plan's workspace and are shared by rs_plan_forward (FiLM rows
  // 0..B-1 for the caller's timesteps) and by every sampler of the plan (rows 0..T-1 for its schedule): whoever wrote them
  // last owns them.  A sampler re-derives them when it is not the owner or when the weights changed since (weights_epoch).
  const void* table_owner = nullptr;
  unsigned long long table_epoch = ~0ull;

  int new_tensor(size_t bytes, bool persistent = false) {
    Tensor t; t.bytes = align_up(bytes, 256); t.persistent = persistent;
    tensors.push_back(t);
    return (int)tensors.size() - 1;
  }
  View make_view(int N, int Hh, int Ww, int C, bool persistent = false) {
    View v; v.N = N; v.H = Hh; v.W = Ww; v.C = C; v.ld = C; v.off = 0;
    v.tens = new_tensor((size_t)N * Hh * Ww * C * 2, persistent);
    return v;
  }
  static View slice(const View& base, int c0, int C) {
    View v = base; v.off = base.off + c0; v.c0 = base.c0 + c0; v.C = C; return v;
  }
  void touch(const View& v, int opi) {
    if (v.tens < 0) return;
    Tensor& t = tensors[v.tens];
    t.first = std::min(t.first, opi); t.last = std::max(t.last, opi);
  }
};

namespace {

struct Builder {
  rs_plan& P;
  rs_engine& E;
  std::vector<Op>* cur;
  size_t stats_off = 0;
  int n_gn = 0;
  struct Writer { int c0; int C; int n0; int N; int list; int op; int win_slots; };
  std::map<int, std::vector<Writer>> writers;      // tensor id -> latest writers by (channel range, image range)
  static bool overlaps(const Writer& w, const View& v, int C) {
    return w.c0 < v.c0 + C && v.c0 < w.c0 + w.C && w.n0 < v.n0 + v.N && v.n0 < w.n0 + w.N;
  }
  static bool inside(const Writer& w, const View& v) {
    return w.c0 >= v.c0 && w.c0 + w.C <= v.c0 + v.C && w.n0 >= v.n0 && w.n0 + w.N <= v.n0 + v.N;
  }
  void note_writer(const View& out, int C, int win_slots = 0) {
    forget_writers(out, C);
    writers[out.tens].push_back({out.c0, C, out.n0, out.N, list_id(), (int)cur->size() - 1, win_slots});
  }
  // the op a writer names: a conv, fused MLP or fused Swin attention (the kinds that note writers)
  Producer& producer(const Writer& w) {
    Op& op = list(w.list)[w.op];
    if (ConvOp* c = std::get_if<ConvOp>(&op)) return *c;
    if (MlpOp* m = std::get_if<MlpOp>(&op)) return *m;
    return payload<SwinOp>(op);
  }
  // producers of every (channel, image) of `in` whose epilogues can deliver GroupNorm statistics (empty: not fusable)
  std::vector<Writer> covering_writers(const View& in) {
    bool fusable = false;
    conv_tile_slots(in.H, in.W, &fusable);
    std::vector<Writer> prod;
    if (fuse_stats && fusable) {
      long long covered = 0;
      auto it = writers.find(in.tens);
      if (it != writers.end())
        for (const Writer& w : it->second)
          if (inside(w, in)) { prod.push_back(w); covered += (long long)w.C * w.N; }
      bool ok = covered == (long long)in.C * in.N;
      for (const Writer& w : prod) ok = ok && producer(w).stat_dst.size() < 2 && w.win_slots == prod[0].win_slots;
      if (!ok) prod.clear();
    }
    return prod;
  }
  // The statistics of a GroupNorm over `in`, with its pair buffer and group-statistics index reserved: from the producers'
  // epilogues when they can deliver them (the consumer is added to their stat_dst), else from gn_stats_kernel in gn_chunks
  // slots, or, with fused_only, none (nullopt)
  std::optional<GnLink> link_stats(const View& in, float eps, bool fused_only) {
    const std::vector<Writer> prod = covering_writers(in);
    if (prod.empty() && fused_only) return std::nullopt;
    GnLink s{in, !prod.empty(), 0, !prod.empty() && prod[0].win_slots, stats_off, n_gn++, eps};
    if (s.win_slots) s.slots = (in.H / 8) * (in.W / 8);
    else if (s.fused) s.slots = conv_tile_slots(in.H, in.W);
    else { int rows; gn_chunks(in.H * in.W, in.N, &s.slots, &rows); }
    stats_off += align_up((size_t)in.N * s.slots * in.C * 2 * sizeof(float), 256);
    for (const Writer& w : prod) producer(w).stat_dst.push_back({s, w.c0 - in.c0});
    return s;
  }
  // the fused kernels run only where the overrides leave the wgmma conv and attention kernels in place
  const bool fuse_mlp = !P.ovr.conv_simt;
  // norm1 + qkv + window attention + proj + residual as one kernel per Swin block (swin_attn_fused.cuh)
  const bool fuse_swin_attn = !P.ovr.conv_simt && !P.ovr.attn_simt;
  const bool fuse_stats = !P.ovr.conv_direct && !P.ovr.conv_simt;
  Builder(rs_plan& p) : P(p), E(*p.e), cur(&p.ops) {}
  int list_id() const { return cur == &P.fe_ops ? 0 : 1; }
  std::vector<Op>& list(int id) { return id == 0 ? P.fe_ops : P.ops; }

  int opi() const { return (int)(P.fe_ops.size() + P.ops.size()); }

  // SiLU twins (UNetModelConv): a tensor whose every value a ResBlockConv or the head also reads through SiLU has a twin
  // tensor of the same layout holding SiLU of it.  Whoever writes a view of such a tensor (conv epilogue, resample) writes
  // the same view of the twin; with_twin() is the one place that decides which tensors have one.
  std::map<int, int> twin_of;                      // tensor id -> its twin's
  View with_twin(const View& v) {
    if (!twin_of.count(v.tens)) twin_of[v.tens] = P.new_tensor(P.tensors[v.tens].bytes);
    return v;
  }
  bool has_twin(const View& v) const { return twin_of.count(v.tens) != 0; }
  View twin(const View& v) const { View t = v; t.tens = twin_of.at(v.tens); return t; }

  // partial: `out` is a partial value that a later op accumulates into (no twin written)
  void conv(const View& in, const std::string& name, int ksize, int stride, int cout, const View* out,
            const View* res, int act, bool out_f32 = false, int pad_lo = 1, int bias_film_off = -1, int film_off = -1,
            bool partial = false) {
    ConvOp op;
    op.d.in = in; op.d.ksize = ksize; op.d.stride = stride; op.d.Cout = cout; op.d.act = act;
    op.d.pad_lo = pad_lo;
    op.bias_film_off = bias_film_off; op.d.bias_per_image = bias_film_off >= 0;
    op.film_off = film_off; op.d.film = film_off >= 0;
    if (out && !out_f32 && !partial && has_twin(*out)) { op.d.silu_out = twin(*out); op.d.has_silu = true; }
    if (out) { op.d.out = *out; op.d.has_out = true; } else op.d.has_out = false;
    if (res) { op.d.res = *res; op.d.has_res = true; }
    op.w_name = name + ".weight"; op.b_name = name + ".bias";
    op.to_f32 = out_f32;
    if (out && !out_f32 && P.ovr.conv_splitk != 1) {       // split-K for layers with too few tiles
      const TileConfig tc = conv_preview_config(P.ovr, in.N, in.H, in.W, in.C, cout, ksize, stride, true);
      if (tc.splitk > 1) {
        op.d.allow_split = true;
        const size_t bytes = (size_t)tc.splitk * in.N * (in.H / stride) * (in.W / stride) * cout * sizeof(float);
        op.split_tens = P.new_tensor(bytes);
        Tensor& tz = P.tensors[op.split_tens];
        tz.first = tz.last = opi();
      }
    }
    const int i = opi();
    P.touch(in, i); if (out) P.touch(*out, i); if (res) P.touch(*res, i);
    if (op.d.has_silu) P.touch(op.d.silu_out, i);
    cur->push_back(std::move(op));
    if (out && !out_f32 && out->tens >= 0) note_writer(*out, cout);   // the latest writer of this (channel, image) range
  }
  void gn(const View& in, const std::string& name, const View& out, int silu, int film_off, float eps = 1e-5f) {
    GnOp op;
    op.d.out = out; op.d.silu = silu; op.d.film_off = film_off;
    op.stats = *link_stats(in, eps, /*fused_only=*/false);
    op.name = name;
    const int i = opi();
    P.touch(in, i); P.touch(out, i);
    cur->push_back(std::move(op));
  }
  void attn(const View& qkv, const View& out, const std::string& blk, int window, int shift) {
    WinAttnOp op; op.qkv = qkv; op.out = out; op.window = window; op.shift = shift; op.simt = P.ovr.attn_simt;
    op.bias_name = blk + ".attn.relative_position_bias_table";
    const int i = opi();
    P.touch(qkv, i); P.touch(out, i);
    cur->push_back(std::move(op));
  }
  void mlp(const View& in, const std::string& name, int E, int Hd, const View& out, const View& res) {
    MlpOp op;
    op.d.in = in; op.d.out = out; op.d.res = res; op.d.has_res = true; op.d.E = E; op.d.Hd = Hd;
    op.name = name;
    const int i = opi();
    P.touch(in, i); P.touch(out, i); P.touch(res, i);
    cur->push_back(std::move(op));
    if (out.tens >= 0) note_writer(out, E);
  }
  // x <- x + proj(window_attention(qkv(norm1(x)))) in one kernel (swin_attn_fused.cuh); false when the statistics of x
  // cannot come from its producers' epilogues
  bool swin_attn(const View& x, const std::string& blk, int heads, int shift) {
    const std::optional<GnLink> norm1 = link_stats(x, 1e-5f, /*fused_only=*/true);
    if (!norm1) return false;
    SwinOp op;
    op.d.x = x; op.d.y = x; op.d.heads = heads; op.d.shift = shift;
    op.blk = blk;
    op.norm1 = *norm1;
    const int i = opi();
    P.touch(x, i);
    cur->push_back(std::move(op));
    if (x.tens >= 0) note_writer(x, x.C, /*win_slots=*/1);
    return true;
  }
  // a writer that delivers no GroupNorm statistics: a consumer of this range takes them from gn_stats_kernel
  void forget_writers(const View& out, int C) {
    auto it = writers.find(out.tens);
    if (it == writers.end()) return;
    auto& ws = it->second;
    ws.erase(std::remove_if(ws.begin(), ws.end(), [&](const Writer& w) { return overlaps(w, out, C); }), ws.end());
  }
  void upsample(const View& in, const View& out, bool pool = false) {
    const int i = opi();
    P.touch(in, i); P.touch(out, i);
    ResampleOp r{in, out, pool};
    if (has_twin(out)) { r.silu = twin(out); r.has_silu = true; P.touch(r.silu, i); }
    cur->push_back(r);
    forget_writers(out, out.C);
  }

  // ResBlock (reference models/unet.py:186-206)
  // updown: 0, or -1 / +1 for a ResBlock with down / up = True: h_upd and x_upd resample the GroupNorm + SiLU output and x
  // (2x2 average pool / nearest 2x, :187-193).  Without scale-shift norm, h + emb_out is in_layers.2's epilogue bias.
  void res_block(const View& x_in, const std::string& p, int cout, const View& out, int updown = 0) {
    const bool ss = E.opt.use_scale_shift_norm != 0;
    View t1 = P.make_view(x_in.N, x_in.H, x_in.W, x_in.C);
    gn(x_in, p + ".in_layers.0", t1, 1, -1);
    View x = x_in;
    if (updown) {
      const int Ho = updown > 0 ? 2 * x_in.H : x_in.H / 2, Wo = updown > 0 ? 2 * x_in.W : x_in.W / 2;
      View t1r = P.make_view(x_in.N, Ho, Wo, x_in.C);
      upsample(t1, t1r, updown < 0);
      t1 = t1r;
      x = P.make_view(x_in.N, Ho, Wo, x_in.C);
      upsample(x_in, x, updown < 0);
    }
    View h1 = P.make_view(x.N, x.H, x.W, cout);
    conv(t1, p + ".in_layers.2", 3, 1, cout, &h1, nullptr, ACT_NONE, false, 1, ss ? -1 : E.film_row_of.at(p));
    View t2 = P.make_view(x.N, x.H, x.W, cout);
    gn(h1, p + ".out_layers.0", t2, 1, ss ? E.film_row_of.at(p) : -1);
    if (x.C != cout) {
      conv(x, p + ".skip_connection", 1, 1, cout, &out, nullptr, ACT_NONE);
      conv(t2, p + ".out_layers.3", 3, 1, cout, &out, &out, ACT_NONE);     // in-place accumulate
    } else {
      conv(t2, p + ".out_layers.3", 3, 1, cout, &out, &x, ACT_NONE);
    }
  }
  // ResBlockConv (reference models/unet.py:984-1004): y = skip(x) + out_conv(SiLU(in_conv(SiLU(x)) + emb_out)), or with
  // scale-shift norm y = skip(x) + out_conv(SiLU(in_conv(SiLU(x))) * (1 + scale) + shift) (out_layers[0] is the SiLU, and
  // no SiLU follows the FiLM).  SiLU(x) is x's twin; in_conv's epilogue adds emb_out as its per-image bias and applies the
  // SiLU (and the FiLM).  updown: h_upd / x_upd resample SiLU(x) and x (:985-990).  out_conv's epilogue writes y and its twin.
  void res_block_conv(const View& x_in, const std::string& p, int cout, const View& out, int updown = 0) {
    const bool ss = E.opt.use_scale_shift_norm != 0;
    const int row = E.film_row_of.at(p);
    View s = twin(x_in);
    View x = x_in;
    if (updown) {
      const int Ho = updown > 0 ? 2 * x_in.H : x_in.H / 2, Wo = updown > 0 ? 2 * x_in.W : x_in.W / 2;
      View sr = P.make_view(x_in.N, Ho, Wo, x_in.C);
      upsample(s, sr, updown < 0);
      s = sr;
      x = P.make_view(x_in.N, Ho, Wo, x_in.C);
      upsample(x_in, x, updown < 0);
    }
    View h = P.make_view(x.N, x.H, x.W, cout);
    conv(s, p + ".in_layers.1", 3, 1, cout, &h, nullptr, ACT_SILU, false, 1, ss ? -1 : row, ss ? row : -1);
    if (x.C != cout) {
      conv(x, p + ".skip_connection", 1, 1, cout, &out, nullptr, ACT_NONE, false, 1, -1, -1, /*partial=*/true);
      conv(h, p + ".out_layers.1", 3, 1, cout, &out, &out, ACT_NONE);     // in-place accumulate
    } else {
      conv(h, p + ".out_layers.1", 3, 1, cout, &out, &x, ACT_NONE);
    }
  }
  // BasicLayer (reference models/swin_transformer.py:427-442) with SwinTransformerBlock.forward (:238-281)
  int basic_layer(const View& x, const std::string& p, int ctor_res, const View& out) {
    const rs_unet_config& c = E.cfg;
    const int Ed = c.swin_embed_dim, hidden = (int)(Ed * c.mlp_ratio);
    const int win = ctor_res <= c.window_size ? ctor_res : c.window_size;
    RS_CHECK((win == 8 || win == 16) && x.H % win == 0 && x.W % win == 0,
             "a " + std::to_string(x.H) + "x" + std::to_string(x.W) + " level with " + std::to_string(win) + "x" + std::to_string(win) +
             " windows: the window-attention kernels cover 8x8 and 16x16 windows that tile the level");
    const int shift_odd = ctor_res <= c.window_size ? 0 : c.window_size / 2;
    View e = P.make_view(x.N, x.H, x.W, Ed);
    if (E.opt.patch_norm) {
      // PatchEmbed.norm (reference models/swin_transformer.py:452-502).  Its output comes from no conv epilogue, so the
      // first block's norm1 takes its statistics from gn_stats_kernel and that block runs the four-launch form
      View e0 = P.make_view(x.N, x.H, x.W, Ed);
      conv(x, p + ".patch_embed.proj", 1, 1, Ed, &e0, nullptr, ACT_NONE);
      gn(e0, p + ".patch_embed.norm", e, 0, -1);
    } else {
      conv(x, p + ".patch_embed.proj", 1, 1, Ed, &e, nullptr, ACT_NONE);
    }
    for (int i = 0; i < c.swin_depth; ++i) {
      const std::string b = p + ".blocks." + std::to_string(i);
      // x = x + proj(attn(qkv(norm1(x)))): one kernel (swin_attn_fused.cuh), or the four-launch sequence
      // (a level with few window pairs is one long serial tile per CTA on a handful of SMs: below swin_fuse_min_pairs
      //  (Overrides) the four small launches, whose prologues overlap through PDL, are faster in the graph)
      const int win_pairs = (x.N * (x.H / win) * (x.W / win) + 1) / 2;
      if (!(fuse_swin_attn && win_pairs >= P.ovr.swin_fuse_min_pairs && swin_attn_supported(Ed, c.swin_heads, x.H, x.W, win) &&
            swin_attn(e, b, c.swin_heads, (i % 2) ? shift_odd : 0))) {
        View n1 = P.make_view(x.N, x.H, x.W, Ed);
        gn(e, b + ".norm1", n1, 0, -1);
        View qkv = P.make_view(x.N, x.H, x.W, 3 * Ed);
        conv(n1, b + ".attn.qkv", 1, 1, 3 * Ed, &qkv, nullptr, ACT_NONE);
        View a = P.make_view(x.N, x.H, x.W, Ed);
        attn(qkv, a, b, win, (i % 2) ? shift_odd : 0);
        conv(a, b + ".attn.proj", 1, 1, Ed, &e, &e, ACT_NONE);              // x = shortcut + attn
      }
      View n2 = P.make_view(x.N, x.H, x.W, Ed);
      gn(e, b + ".norm2", n2, 0, -1);
      if (fuse_mlp && mlp_supported(Ed, hidden, x.H, x.W, x.N)) {
        mlp(n2, b + ".mlp", Ed, hidden, e, e);                            // x = x + fc2(gelu(fc1(n2))), one kernel
      } else {
        View f = P.make_view(x.N, x.H, x.W, hidden);
        conv(n2, b + ".mlp.fc1", 1, 1, hidden, &f, nullptr, ACT_GELU);
        conv(f, b + ".mlp.fc2", 1, 1, Ed, &e, &e, ACT_NONE);              // x = x + mlp
      }
    }
    if (E.opt.patch_norm) {
      // PatchUnEmbed.norm (:504-527), written into the block's destination (possibly a channel slice of a concat buffer)
      View u = P.make_view(x.N, x.H, x.W, x.C);
      conv(e, p + ".patch_unembed.proj", 1, 1, x.C, &u, nullptr, ACT_NONE);
      gn(u, p + ".patch_unembed.norm", out, 0, -1);
      forget_writers(out, x.C);
    } else {
      conv(e, p + ".patch_unembed.proj", 1, 1, x.C, &out, nullptr, ACT_NONE);
    }
    return 0;
  }

  // AttentionBlock of UNetModel (reference models/unet.py:257-263): out = x + proj_out(attention(qkv(norm(x)))) as four
  // launches; norm takes its statistics from x's producers, proj_out's epilogue delivers those of out to its consumers
  void unet_attn_block(const View& x, const std::string& p, int heads, const View& out) {
    View n = P.make_view(x.N, x.H, x.W, x.C);
    gn(x, p + ".norm", n, 0, -1);
    View qkv = P.make_view(x.N, x.H, x.W, 3 * x.C);
    conv(n, p + ".qkv", 1, 1, 3 * x.C, &qkv, nullptr, ACT_NONE);
    View a = P.make_view(x.N, x.H, x.W, x.C);
    UnetAttnDesc op;
    op.qkv = qkv; op.out = a; op.heads = heads; op.new_order = E.um.use_new_attention_order != 0;
    const int i = opi();
    P.touch(qkv, i); P.touch(a, i);
    cur->push_back(std::move(op));
    conv(a, p + ".proj_out", 1, 1, x.C, &out, &x, ACT_NONE);
  }

  int run_block(View h, const std::string& prefix, const std::vector<Layer>& layers, const View& dest, View* result) {
    for (size_t j = 0; j < layers.size(); ++j) {
      const Layer& L = layers[j];
      const std::string p = prefix + "." + std::to_string(j);
      const bool last = (j + 1 == layers.size());
      // an output inside the block: with a twin when a ResBlockConv reads it next (block outputs are the caller's dest)
      auto inner = [&](int c) {
        const View v = P.make_view(h.N, h.H, h.W, c);
        const int nk = last ? -1 : layers[j + 1].kind;
        return E.conv_blocks && (nk == L_RES || nk == L_RES_DOWN || nk == L_RES_UP) ? with_twin(v) : v;
      };
      View out;
      if (L.kind == L_CONV) {
        out = last ? dest : inner(L.b);
        conv(h, p, 3, 1, L.b, &out, nullptr, ACT_NONE);
      } else if (L.kind == L_RES && E.conv_blocks) {
        out = last ? dest : inner(L.b);
        res_block_conv(h, p, L.b, out);
      } else if (L.kind == L_RES) {
        out = last ? dest : P.make_view(h.N, h.H, h.W, L.b);
        res_block(h, p, L.b, out);
      } else if (L.kind == L_SWIN) {
        out = last ? dest : P.make_view(h.N, h.H, h.W, h.C);
        int rc = basic_layer(h, p, L.b, out); if (rc) return rc;
      } else if (L.kind == L_ATTN) {
        out = last ? dest : P.make_view(h.N, h.H, h.W, h.C);
        unet_attn_block(h, p, L.b, out);
      } else if (L.kind == L_RES_DOWN || L.kind == L_RES_UP) {     // always the last layer of its block
        out = dest;
        if (E.conv_blocks) res_block_conv(h, p, L.a, out, L.kind == L_RES_DOWN ? -1 : 1);
        else res_block(h, p, L.a, out, L.kind == L_RES_DOWN ? -1 : 1);
      } else if (L.kind == L_DOWN) {
        out = dest;
        if (E.opt.conv_resample) conv(h, p + ".op", 3, 2, L.a, &out, nullptr, ACT_NONE);
        else upsample(h, out, /*pool=*/true);
      } else if (!E.opt.conv_resample) {
        out = dest;
        upsample(h, out);
      } else {
        View u = P.make_view(h.N, 2 * h.H, 2 * h.W, h.C);
        upsample(h, u);
        out = dest;
        conv(u, p + ".conv", 3, 1, L.a, &out, nullptr, ACT_NONE);
      }
      h = out;
    }
    *result = h;
    return 0;
  }
};

// Workspace layout shared by the denoiser plan and the VQ-GAN plans (vq.inc): fixed regions, then persistent tensors,
// then liveness-packed temporaries.  `state_bytes` = one fp32 latent / output image; the denoiser keeps two (x_t, model out).
int finish_layout(rs_plan& P, Builder& b, size_t state_bytes, bool unet) {
  rs_engine& E = *P.e;
  const rs_unet_config& c = E.cfg;
  const int B = P.B;
  P.max_rows = std::max(B, 64);
  size_t off = 0;
  auto region = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  if (unet) {
    P.off_tables = region(kStepRows * 1024 * sizeof(float));   // the sampler's step tables (StepParams::row), <= 1024 steps each
    P.off_tsteps = region((size_t)P.max_rows * sizeof(float));
    P.off_emb_sin = region((size_t)P.max_rows * c.model_channels * sizeof(float));
    P.off_emb_mid = region((size_t)P.max_rows * E.time_dim() * sizeof(float));
    P.off_emb_vec = region((size_t)P.max_rows * E.time_dim() * sizeof(float));
    P.off_film = region((size_t)P.max_rows * E.film_rows * sizeof(float));
  }
  P.stats_bytes = b.stats_off;
  P.off_stats = region(P.stats_bytes);
  P.n_gn = b.n_gn;
  P.off_gstat = region((size_t)P.n_gn * B * 32 * 2 * sizeof(float));
  P.off_counters = region((size_t)P.n_gn * B * sizeof(unsigned int));
  // sampler state: x_t (fp32), model output / pred_xstart (fp32)
  const size_t lat = state_bytes;
  P.off_state = region(2 * align_up(lat, 256));
  // persistent tensors first, then liveness-packed temporaries (RS_NO_REUSE=1 keeps every tensor
  // alive for the whole forward so that rs_plan_probe can read any block output afterwards)
  if (P.ovr.no_reuse) for (Tensor& tz : P.tensors) tz.persistent = true;
  for (Tensor& tz : P.tensors) if (tz.persistent) tz.off = region(tz.bytes);
  P.off_temps = off;
  {
    struct Live { size_t off, bytes; int last; };
    std::vector<Live> live;
    std::vector<int> order;
    for (int i = 0; i < (int)P.tensors.size(); ++i) if (!P.tensors[i].persistent && P.tensors[i].last >= 0) order.push_back(i);
    std::stable_sort(order.begin(), order.end(), [&](int a, int bb) { return P.tensors[a].first < P.tensors[bb].first; });
    size_t high = 0;
    for (int id : order) {
      Tensor& tz = P.tensors[id];
      live.erase(std::remove_if(live.begin(), live.end(), [&](const Live& l) { return l.last < tz.first; }), live.end());
      std::sort(live.begin(), live.end(), [](const Live& a, const Live& bb) { return a.off < bb.off; });
      size_t pos = 0;
      for (const Live& l : live) {
        if (pos + tz.bytes <= l.off) break;
        pos = std::max(pos, l.off + l.bytes);
      }
      tz.off = P.off_temps + pos;
      live.push_back({pos, tz.bytes, tz.last});
      high = std::max(high, pos + tz.bytes);
    }
    P.temps_bytes = high;
  }
  P.workspace_bytes = align_up(P.off_temps + P.temps_bytes, 256);
  return 0;
}

int build_plan(rs_plan& P) {
  rs_engine& E = *P.e;
  const rs_unet_config& c = E.cfg;
  Topology topo = build_topology(E);
  Builder b(P);
  const int B = P.B;

  // ---- feature extractor (reference models/unet.py:689-702), hoisted out of the sampling loop ----
  const int fes = E.fe_stages();
  P.lqH = (P.H << fes) * E.lq_factor(); P.lqW = (P.W << fes) * E.lq_factor();
  if (fes > 0) {
    b.cur = &P.fe_ops;
    P.fe_cpad = 8;
    P.fe_in = P.make_view(B, P.lqH, P.lqW, P.fe_cpad, true);
    View cur = P.fe_in;
    int bc = 16;
    for (int st = 0; st < fes; ++st) {
      View a = P.make_view(B, cur.H, cur.W, bc, true);
      b.conv(cur, "feature_extractor." + std::to_string(3 * st), 3, 1, bc, &a, nullptr, ACT_SILU);
      View d = P.make_view(B, cur.H / 2, cur.W / 2, 2 * bc, true);
      b.conv(a, "feature_extractor." + std::to_string(3 * st + 2) + ".op", 3, 2, 2 * bc, &d, nullptr, ACT_NONE);
      cur = d; bc *= 2;
    }
    P.lq_feat = cur;
    b.cur = &P.ops;
  }

  // ---- main body -----------------------------------------------------------------------------
  const int cin = c.in_channels + E.lq_feat_ch();
  P.cin_pad = (cin + 7) / 8 * 8;
  P.xin = P.make_view(B, P.H, P.W, P.cin_pad, true);

  // concat buffers of the decoder: output block j reads cat([h, hs[n_in-1-j]])
  const int n_in = (int)topo.input_blocks.size();
  const int n_out = (int)topo.output_blocks.size();
  RS_CHECK(n_in == n_out, "encoder/decoder block counts differ");
  // resolutions of the encoder outputs
  std::vector<int> in_h(n_in), in_w(n_in);
  {
    int hh = P.H, ww = P.W;
    for (int i = 0; i < n_in; ++i) {
      for (const Layer& L : topo.input_blocks[i]) if (L.kind == L_DOWN || L.kind == L_RES_DOWN) { hh /= 2; ww /= 2; }
      in_h[i] = hh; in_w[i] = ww;
    }
  }
  std::vector<View> cat(n_out);
  for (int j = 0; j < n_out; ++j) {
    const int k = n_in - 1 - j;
    const int ctot = topo.output_blocks[j][0].a;       // ch + ich
    cat[j] = P.make_view(B, in_h[k], in_w[k], ctot);
    if (E.conv_blocks) b.with_twin(cat[j]);            // read by a ResBlockConv: every slice writer also writes SiLU of it
  }
  // encoder
  View h = P.xin;
  for (int i = 0; i < n_in; ++i) {
    const int j = n_in - 1 - i;
    const int ich = topo.in_block_ch[i];
    View dest = rs_plan::slice(cat[j], cat[j].C - ich, ich);
    // the input view of the first conv must expose the padded channel count (weights are zero-padded)
    View hin = h;
    int rc = b.run_block(hin, "input_blocks." + std::to_string(i), topo.input_blocks[i], dest, &h);
    if (rc) return rc;
    P.block_out["input_blocks." + std::to_string(i)] = h;
  }
  // middle: writes into the h-slice of cat[0]
  {
    View dest = rs_plan::slice(cat[0], 0, cat[0].C - topo.in_block_ch[n_in - 1]);
    int rc = b.run_block(h, "middle_block", topo.middle, dest, &h); if (rc) return rc;
    P.block_out["middle_block"] = h;
  }
  // decoder
  View final_h;
  for (int j = 0; j < n_out; ++j) {
    View dest;
    if (j + 1 < n_out) {
      const int ich_next = topo.in_block_ch[n_in - 2 - j];
      dest = rs_plan::slice(cat[j + 1], 0, cat[j + 1].C - ich_next);
    } else {
      const Layer& L0 = topo.output_blocks[j][0];
      dest = P.make_view(B, cat[j].H, cat[j].W, L0.b);
      if (E.conv_blocks) b.with_twin(dest);            // the head reads SiLU(h)
    }
    int rc = b.run_block(cat[j], "output_blocks." + std::to_string(j), topo.output_blocks[j], dest, &h);
    if (rc) return rc;
    P.block_out["output_blocks." + std::to_string(j)] = h;
    final_h = h;
  }
  // head (reference models/unet.py:859-863,894; UNetModelConv :1148-1151: conv3x3(SiLU(h)))
  if (E.conv_blocks) {
    b.conv(b.twin(final_h), "out.1", 3, 1, c.out_channels, nullptr, nullptr, ACT_NONE, /*out_f32=*/true);
  } else {
    View t = P.make_view(B, final_h.H, final_h.W, final_h.C);
    b.gn(final_h, "out.0", t, 1, -1);
    b.conv(t, "out.2", 3, 1, c.out_channels, nullptr, nullptr, ACT_NONE, /*out_f32=*/true);
  }

  return finish_layout(P, b, (size_t)B * std::max(c.in_channels, c.out_channels) * P.H * P.W * sizeof(float), true);
}

void resolve(rs_plan& P, View& v) {
  if (v.tens >= 0) v.ptr = reinterpret_cast<__half*>(P.ws + P.tensors[v.tens].off) + v.off;
}

// statistics destination of a producer: the consuming GroupNorm's pair buffer (+ group statistics / arrival counters)
// Who reduces the (mean, M2) pairs to the image's 32 (mean, rstd)?
//   * few tile slots (the denoiser's maps, <= 32 slots): every consumer CTA combines them itself — a finalisation step on
//     the producer's tail sits on every producer CTA;
//   * many slots (more than kGnFinalizeSlots: the VQ-GAN's 128x128 / 256x256 maps): gn_finalize_kernel, a
//     small launch in front of the consumer, or, for a GroupNorm without a fusable producer, the last gn_stats_kernel CTA
//     of each image (arrival counters).  (The last producer CTA of an image would do it at the cost of a counter round
//     trip on every tile, and on a persistent conv the CTAs all finish together, so ONE of them would reduce every image.)
constexpr int kGnFinalizeSlots = 64;
bool gn_finalizes(const GnLink& g) {
  return g.slots > kGnFinalizeSlots && !g.win_slots;      // (the fused Swin attention kernel delivers pairs only)
}
GnSink make_sink(rs_plan& P, const GnLink& g, int coff, bool consumer = false) {
  GnSink s{};
  s.part = reinterpret_cast<float*>(P.ws + P.off_stats + g.stats_off);
  if (consumer && gn_finalizes(g)) {
    s.gstat = reinterpret_cast<float*>(P.ws + P.off_gstat) + (size_t)g.gn_index * P.B * 64;
    s.counter = reinterpret_cast<unsigned int*>(P.ws + P.off_counters) + (size_t)g.gn_index * P.B;
  }
  s.cstride = g.in.C; s.coff = coff; s.expected = (unsigned)(g.slots * g.in.C); s.eps = g.eps;
  return s;
}
// the statistics sinks of a producer's epilogue: one per consumer it delivers to
void bind_sinks(rs_plan& P, const Producer& pr, GnSink (&sink)[2]) {
  for (int i = 0; i < 2; ++i)
    sink[i] = i < (int)pr.stat_dst.size() ? make_sink(P, pr.stat_dst[i].to, pr.stat_dst[i].coff) : GnSink{};
}

int bind_ops(rs_plan& P, std::vector<Op>& ops) {
  rs_engine& E = *P.e;
  for (Op& op : ops) {
    int rc = 0, launches = 1;
    switch (kind_of(op)) {
      case OP_CONV: {
        ConvOp& c = payload<ConvOp>(op);
        ConvDesc& d = c.d;
        bind_sinks(P, c, d.sink);
        resolve(P, d.in); if (d.has_out) resolve(P, d.out); if (d.has_res) resolve(P, d.res);
        if (d.has_silu) resolve(P, d.silu_out);
        if (!c.in_param.empty()) {          // the "pixels" are the rows of a weight matrix of the arena
          const Param* wp = E.find(c.in_param);
          RS_CHECK(wp != nullptr && wp->ipad == d.in.ld, "missing / mismatching parameter " + c.in_param);
          d.in.ptr = E.at<__half>(c.in_param);
        }
        if (c.w_is_view) {                  // the "weights" are an activation tensor [Cout rows][K], K-major
          resolve(P, c.w_view);
          d.wt = c.w_view.ptr; d.ipad = c.w_view.ld;
          d.bias = c.b_name.empty() ? nullptr : E.at<float>(c.b_name);
        } else {
          d.wt = E.packed(c.w_name, &d.ipad); d.bias = E.at<float>(c.b_name);
          RS_CHECK(d.wt != nullptr, "missing parameter " + c.w_name);
        }
        d.out_f32 = c.to_f32 ? P.out_f32 : nullptr;
        d.partial = c.split_tens >= 0 ? reinterpret_cast<float*>(P.ws + P.tensors[c.split_tens].off) : nullptr;
        // the first conv reads the channel-padded packed input: expose the padded width to the kernel
        if (d.in.C < d.ipad && d.in.ld >= d.ipad && d.in.tens == P.xin.tens) d.in.C = d.ipad;
        if (d.in.C < d.ipad && P.fe_in.tens >= 0 && d.in.tens == P.fe_in.tens) d.in.C = d.ipad;
        rc = conv_finalize(d, P.ovr); if (rc) return rc;
        RS_CHECK(d.prm.splitk == 1 || (size_t)d.prm.splitk * d.prm.Nimg * d.prm.Hout * d.prm.Wout * d.Cout * sizeof(float) <=
                                       P.tensors[c.split_tens].bytes, "split-K scratch of " + c.w_name + " too small for the split chosen");
        launches = d.prm.splitk > 1 ? 2 : 1;
        break;
      }
      case OP_GN: {
        GnOp& g = payload<GnOp>(op);
        GnDesc& d = g.d;
        d.in = g.stats.in; d.fused = g.stats.fused; d.slots = g.stats.slots; d.eps = g.stats.eps;
        resolve(P, d.in); resolve(P, d.out);
        d.gamma = E.at<float>(g.name + ".weight"); d.beta = E.at<float>(g.name + ".bias");
        RS_CHECK(d.gamma && d.beta, "missing GroupNorm parameters " + g.name);
        const GnSink sk = make_sink(P, g.stats, 0, true);
        d.part = sk.part; d.gstat = sk.gstat; d.counter = sk.counter;
        d.finalize_kernel = d.fused && gn_finalizes(g.stats);
        launches = (d.fused ? 1 : 2) + (d.finalize_kernel ? 1 : 0);
        break;
      }
      case OP_ATTN: {
        WinAttnOp& a = payload<WinAttnOp>(op);
        resolve(P, a.qkv); resolve(P, a.out);
        a.bias = E.at<float>(a.bias_name);
        RS_CHECK(a.bias != nullptr, "missing " + a.bias_name);
        break;
      }
      case OP_UPSAMPLE: {
        ResampleOp& r = payload<ResampleOp>(op);
        resolve(P, r.in); resolve(P, r.out);
        if (r.has_silu) resolve(P, r.silu);
        break;
      }
      case OP_MLP: {
        MlpOp& mo = payload<MlpOp>(op);
        MlpDesc& m = mo.d;
        resolve(P, m.in); resolve(P, m.out); resolve(P, m.res);
        int ld1 = 0, ld2 = 0;
        m.w1 = E.packed(mo.name + ".fc1.weight", &ld1); m.b1 = E.at<float>(mo.name + ".fc1.bias");
        m.w2 = E.packed(mo.name + ".fc2.weight", &ld2); m.b2 = E.at<float>(mo.name + ".fc2.bias");
        RS_CHECK(m.w1 && m.w2 && m.b1 && m.b2, "missing MLP parameters " + mo.name + ".fc1.weight");
        RS_CHECK(ld1 == m.E && ld2 == m.Hd, "MLP weight padding");
        bind_sinks(P, mo, m.sink);
        rc = mlp_finalize(m);
        break;
      }
      case OP_SOFTMAX: resolve(P, payload<SoftmaxOp>(op).view); rc = softmax_rows_check(softmax_params(payload<SoftmaxOp>(op))); break;
      case OP_SWIN_ATTN: {
        SwinOp& so = payload<SwinOp>(op);
        SwinAttnDesc& w = so.d;
        resolve(P, w.x); resolve(P, w.y);
        const std::string& b = so.blk;
        w.wqkv = E.packed(b + ".attn.qkv.weight", &w.wqkv_ld); w.bqkv = E.at<float>(b + ".attn.qkv.bias");
        w.wproj = E.packed(b + ".attn.proj.weight", &w.wproj_ld); w.bproj = E.at<float>(b + ".attn.proj.bias");
        w.relbias = E.at<float>(b + ".attn.relative_position_bias_table");
        w.gamma = E.at<float>(b + ".norm1.weight"); w.beta = E.at<float>(b + ".norm1.bias");
        RS_CHECK(w.wqkv && w.wproj && w.bqkv && w.bproj && w.relbias && w.gamma && w.beta, "missing attention parameters of " + b);
        const GnSink sk = make_sink(P, so.norm1, 0);
        w.gn_part = sk.part; w.gn_slots = so.norm1.slots;
        bind_sinks(P, so, w.sink);
        rc = swin_attn_finalize(w);
        break;
      }
      case OP_VQ_ATTN: {
        VqAttnDesc& a = payload<VqAttnDesc>(op);
        resolve(P, a.q); resolve(P, a.k); resolve(P, a.v); resolve(P, a.out);
        rc = vq_attn_finalize(a);
        break;
      }
      case OP_UNET_ATTN: {
        UnetAttnDesc& a = payload<UnetAttnDesc>(op);
        resolve(P, a.qkv); resolve(P, a.out);
        rc = unet_attn_finalize(a);
        break;
      }
    }
    if (rc) return rc;
    P.launches += launches;
  }
  return 0;
}

struct Prof {
  std::vector<cudaEvent_t> ev;     // a pair per op run
  int used = 0;
  cudaEvent_t get() {
    if (used == (int)ev.size()) { cudaEvent_t e; cudaEventCreate(&e); ev.push_back(e); }
    return ev[used++];
  }
  ~Prof() { for (cudaEvent_t e : ev) cudaEventDestroy(e); }
};

// ops [first, last) of an op list
int run_op_range(rs_plan& P, const Op* first, const Op* last, const float* film_base, long long film_sN, cudaStream_t st,
                 Prof* prof = nullptr) {
  for (const Op* it = first; it != last; ++it) {
    const Op& op = *it;
    int rc = 0;
    if (prof) cudaEventRecord(prof->get(), st);
    switch (kind_of(op)) {
      case OP_CONV: {
        const ConvOp& c = payload<ConvOp>(op);
        if (c.bias_film_off < 0 && c.film_off < 0) { rc = conv_launch(c.d, st); break; }
        ConvDesc d = c.d;               // bias / FiLM = this launch's FiLM-table row(s), resolved like a GroupNorm's film
        if (c.bias_film_off >= 0) {
          const float* row = film_base + c.bias_film_off;
          if (d.prm.bias) { d.prm.bias = row; d.prm.bias_sN = (int)film_sN; }
          if (d.prm.splitk > 1) { d.red.bias = row; d.red.bias_sN = (int)film_sN; }
        }
        if (c.film_off >= 0) {
          const float* row = film_base + c.film_off;
          if (d.prm.splitk > 1) { d.red.film = row; d.red.film_sN = (int)film_sN; }
          else { d.prm.film = row; d.prm.film_sN = (int)film_sN; }
        }
        rc = conv_launch(d, st);
        break;
      }
      case OP_GN: {
        GnDesc g = payload<GnOp>(op).d;
        if (g.film_off >= 0) { g.film = film_base + g.film_off; g.film_sN = film_sN; }
        rc = gn_launch(g, st);
        break;
      }
      case OP_MLP: rc = mlp_launch(payload<MlpOp>(op).d, st); break;
      case OP_SWIN_ATTN: rc = swin_attn_launch(payload<SwinOp>(op).d, st); break;
      case OP_VQ_ATTN: rc = vq_attn_launch(payload<VqAttnDesc>(op), st); break;
      case OP_UNET_ATTN: rc = unet_attn_launch(payload<UnetAttnDesc>(op), st); break;
      case OP_ATTN: {
        const WinAttnOp& a = payload<WinAttnOp>(op);
        rc = attn_launch(a.qkv, a.out, a.bias, P.e->cfg.swin_heads, P.e->cfg.swin_embed_dim, a.window, a.shift, a.simt, st);
        break;
      }
      case OP_SOFTMAX: {
        const SoftmaxParams sp = softmax_params(payload<SoftmaxOp>(op));
        (void)launch_k(softmax_rows_kernel, dim3((unsigned)sp.rows), dim3(256), (size_t)0, st, sp);
        if (cudaGetLastError() != cudaSuccess) rc = fail(-2, "softmax launch failed");
        break;
      }
      case OP_UPSAMPLE: {
        const ResampleOp& r = payload<ResampleOp>(op);
        UpsampleParams u{r.in.ptr, r.in.sN(), r.in.ld, r.out.ptr, r.out.sN(), r.out.ld, r.in.N, r.in.H, r.in.W, r.in.C};
        if (r.has_silu) { u.s = r.silu.ptr; u.s_sN = r.silu.sN(); u.s_ld = r.silu.ld; }
        const long long total = (long long)u.N * (r.pool ? u.H * u.W / 4 : 4 * u.H * u.W) * (u.C / 8);
        (void)launch_k(r.pool ? avgpool2x2_kernel : upsample2x_kernel,
                       dim3((unsigned)std::min<long long>((total + 255) / 256, num_sms() * 16)), dim3(256), (size_t)(0), st, u);
        if (cudaGetLastError() != cudaSuccess) rc = fail(-2, "resample launch failed");
        break;
      }
    }
    if (prof) cudaEventRecord(prof->get(), st);
    if (rc) return rc;
  }
  return 0;
}

int run_ops(rs_plan& P, const std::vector<Op>& ops, const float* film_base, long long film_sN, cudaStream_t st,
            Prof* prof = nullptr) {
  return run_op_range(P, ops.data(), ops.data() + ops.size(), film_base, film_sN, st, prof);
}

// timestep embedding -> time_embed MLP -> all emb_layers at once, for `rows` timesteps
int run_embedding(rs_plan& P, const float* tsteps, int rows, cudaStream_t st) {
  rs_engine& E = *P.e;
  const int mc = E.cfg.model_channels, K = E.time_dim();
  float* sinb = reinterpret_cast<float*>(P.ws + P.off_emb_sin);
  float* mid = reinterpret_cast<float*>(P.ws + P.off_emb_mid);
  float* vec = reinterpret_cast<float*>(P.ws + P.off_emb_vec);
  float* film = reinterpret_cast<float*>(P.ws + P.off_film);
  const int half = mc / 2;
  (void)launch_k(timestep_embedding_kernel, dim3((rows * half + 127) / 128), dim3(128), (size_t)(0), st, tsteps, sinb, rows, mc);
  auto lin = [&](const float* x, const __half* W, const float* bias, float* out, int Kin, int O, int si, int so) {
    const long long warps = (long long)rows * O;
    (void)launch_k(linear_small_kernel, dim3((unsigned)((warps * 32 + 255) / 256)), dim3(256), (size_t)(0), st, x, W, bias, out, rows, Kin, O, si, so);
  };
  const Param* w0 = E.find("time_embed.0.weight");
  RS_CHECK(w0 && w0->ipad == mc, "time_embed.0 layout");
  lin(sinb, E.at<__half>("time_embed.0.weight"), E.at<float>("time_embed.0.bias"), mid, mc, K, 0, 1);   // Linear -> SiLU
  lin(mid, E.at<__half>("time_embed.2.weight"), E.at<float>("time_embed.2.bias"), vec, K, K, 0, 0);
  lin(vec, reinterpret_cast<__half*>(E.arena + E.film_w_off), reinterpret_cast<float*>(E.arena + E.film_b_off), film,
      K, E.film_rows, 1, 0);                                                                              // SiLU -> Linear
  RS_CUDA_OK(cudaGetLastError());
  return 0;
}

int pack_lq_and_input(rs_plan& P, const float* x, const float* lq, const float* mask, const float* scale_tab,
                      int scale_idx, cudaStream_t st) {
  rs_engine& E = *P.e;
  const rs_unet_config& c = E.cfg;
  const long long npix = (long long)P.B * P.H * P.W;
  PackInputParams pp{};
  pp.x = x; pp.Cx = c.in_channels; pp.scale_tab = scale_tab; pp.scale_idx = scale_idx;
  pp.out = P.xin.ptr; pp.Cpad = P.cin_pad; pp.N = P.B; pp.HW = P.H * P.W;
  pp.zero_ptr = reinterpret_cast<unsigned int*>(P.ws + P.off_counters); pp.zero_n = P.n_gn * P.B;
  if (E.fe_stages() > 0) {
    RS_CHECK(!c.cond_mask || mask != nullptr, "this model is mask-conditioned: mask must be given");
    PackImageParams ip{lq, 3, c.cond_mask ? mask : nullptr, c.cond_mask ? 1 : 0, P.fe_in.ptr, P.fe_cpad, P.B, P.lqH * P.lqW};
    const long long lpix = (long long)P.B * P.lqH * P.lqW;
    (void)launch_k(pack_image_kernel, dim3((unsigned)((lpix + 255) / 256)), dim3(256), (size_t)(0), st, ip);
    int rc = run_ops(P, P.fe_ops, nullptr, 0, st); if (rc) return rc;
    pp.lq_nhwc = P.lq_feat.ptr; pp.lq_ld = P.lq_feat.ld; pp.Cl = P.lq_feat.C;
  } else {
    // no feature extractor: cat([x, lq, mask]) straight into the packed input (reference models/unet.py:876-882); a
    // UNetModel's lq at twice the latent size goes through pixel_unshuffle(lq, 2) on the way (:569-573)
    RS_CHECK(!c.cond_mask || mask != nullptr, "this model is mask-conditioned: mask must be given");
    RS_CHECK(!E.unetmodel || mask == nullptr, "UNetModel.forward takes no mask");
    pp.lq_nchw = lq; pp.Cl = E.unetmodel ? E.lq_feat_ch() : 3;
    pp.mask_nchw = c.cond_mask ? mask : nullptr;
    pp.lq_unshuffle = E.lq_factor() == 2; pp.W = P.W;
  }
  (void)launch_k(pack_input_kernel, dim3((unsigned)((npix + 255) / 256)), dim3(256), (size_t)(0), st, pp);
  RS_CUDA_OK(cudaGetLastError());
  return 0;
}

// A plan runs on the device it was bound on: its workspace, TMA descriptors and the engine's
// arena all belong to that device.  Every run entry point checks the current device first.
int check_plan_device(const rs_plan& P) {
  int dev = -1;
  RS_CUDA_OK(cudaGetDevice(&dev));
  if (dev != P.device)
    return fail(-1, "plan was bound on cuda:" + std::to_string(P.device) + " but cuda:" + std::to_string(dev) +
                    " is current: a plan runs on the device it was bound on");
  return 0;
}

// One forward of the denoiser on the caller's inputs: FiLM rows 0..B-1 for its timesteps, the packed input, the op list
// (with a CUDA-event pair around every op when prof is given)
int run_forward(rs_plan& P, const float* x, const float* timesteps, const float* lq, const float* mask, cudaStream_t st,
                Prof* prof = nullptr) {
  int rc = check_plan_device(P); if (rc) return rc;
  P.table_owner = nullptr;                       // FiLM rows 0..B-1 are overwritten below
  rc = run_embedding(P, timesteps, P.B, st); if (rc) return rc;
  rc = pack_lq_and_input(P, x, lq, mask, nullptr, 0, st); if (rc) return rc;
  return run_ops(P, P.ops, reinterpret_cast<const float*>(P.ws + P.off_film), P.e->film_rows, st, prof);
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

int rs_version(void) { return 100; }
const char* rs_last_error(void) { return g_last_error.c_str(); }

int rs_unet_create_ex(const rs_unet_config* cfg, const rs_unet_options* opts, rs_engine** out) {
  RS_CHECK(cfg && opts && out, "null argument");
  RS_CHECK(cfg->n_levels >= 1 && cfg->n_levels <= RS_MAX_LEVELS, "n_levels");
  RS_CHECK(cfg->swin_heads > 0 && (cfg->swin_embed_dim == cfg->swin_heads * 32 || cfg->swin_embed_dim == cfg->swin_heads * 64),
           "head_dim (swin_embed_dim / heads) must be 32 or 64: the window-attention kernels are instantiated for those");
  RS_CHECK(cfg->window_size == 8 || cfg->window_size == 16,
           "window_size must be 8 or 16: the window-attention kernels are instantiated for 8x8 and 16x16 windows");
  RS_CHECK(cfg->model_channels % 32 == 0 && cfg->swin_embed_dim % 32 == 0, "GroupNorm32 needs channels % 32 == 0");
  RS_CHECK(cfg->lq_size >= cfg->image_size, "lq_size < image_size is not covered");
  for (int v : {opts->use_scale_shift_norm, opts->resblock_updown, opts->conv_resample, opts->patch_norm})
    RS_CHECK(v == 0 || v == 1, "rs_unet_options fields are 0 or 1");
  auto e = std::make_unique<rs_engine>();
  e->cfg = *cfg;
  e->opt = *opts;
  int rc = build_inventory(*e); if (rc) return rc;
  *out = e.release();
  return 0;
}
int rs_unet_create(const rs_unet_config* cfg, rs_engine** out) {
  const rs_unet_options shipped{1, 0, 1, 0};
  return rs_unet_create_ex(cfg, &shipped, out);
}
// The channels of x of a UNetModel / UNetModelConv (x and lq concatenated): out_channels, or with a learned variance
// (learn_sigma: the model outputs the mean, then as many variance values) out_channels / 2; lq adds 3 channels at the
// latent size or 12 at twice it.  Where both readings fit (in 21, out 18) the fixed-variance one wins.  0: neither fits.
static int unet_x_channels(int in, int out) {
  if (out > 0 && (in - out == 3 || in - out == 12)) return out;
  if (out > 0 && out % 2 == 0 && (in - out / 2 == 3 || in - out / 2 == 12)) return out / 2;
  return 0;
}
static const char* const kUnetChannelRule =
    "in_channels must be out_channels + 3 (lq at the latent size) or out_channels + 12 (lq at twice the latent size, "
    "pixel_unshuffle): x has out_channels channels and lq is a 3-channel image; or, with a learned variance (even "
    "out_channels), out_channels / 2 + 3 or out_channels / 2 + 12: x has out_channels / 2 channels";
int rs_unetmodel_create(const rs_unetmodel_config* cfg, const rs_unet_options* opts, rs_engine** out) {
  RS_CHECK(cfg && opts && out, "null argument");
  RS_CHECK(cfg->n_levels >= 1 && cfg->n_levels <= RS_MAX_LEVELS && cfg->n_attn >= 0 && cfg->n_attn <= RS_MAX_LEVELS, "n_levels / n_attn");
  RS_CHECK(opts->patch_norm == 0, "UNetModel has no patch norm: rs_unet_options.patch_norm must be 0");
  for (int v : {opts->use_scale_shift_norm, opts->resblock_updown, opts->conv_resample})
    RS_CHECK(v == 0 || v == 1, "rs_unet_options fields are 0 or 1");
  RS_CHECK(cfg->use_new_attention_order == 0 || cfg->use_new_attention_order == 1, "use_new_attention_order is 0 or 1");
  const int x_ch = unet_x_channels(cfg->in_channels, cfg->out_channels);
  RS_CHECK(x_ch > 0, kUnetChannelRule);
  RS_CHECK(cfg->num_head_channels == -1 || cfg->num_head_channels > 0, "num_head_channels is -1 or positive");
  RS_CHECK(cfg->num_head_channels != -1 || cfg->num_heads > 0, "num_heads must be positive");
  RS_CHECK(cfg->model_channels > 0 && cfg->model_channels % 32 == 0, "GroupNorm32 needs model_channels % 32 == 0");
  for (int l = 0; l < cfg->n_levels; ++l)
    RS_CHECK(cfg->channel_mult[l] > 0 && cfg->num_res_blocks[l] >= 0, "channel_mult / num_res_blocks");
  auto e = std::make_unique<rs_engine>();
  e->unetmodel = true;
  e->um = *cfg;
  e->opt = *opts;
  rs_unet_config& c = e->cfg;
  std::memset(&c, 0, sizeof(c));
  c.image_size = cfg->image_size; c.in_channels = x_ch; c.model_channels = cfg->model_channels;
  c.out_channels = cfg->out_channels; c.n_levels = cfg->n_levels; c.n_attn = cfg->n_attn; c.lq_size = cfg->image_size;
  for (int l = 0; l < RS_MAX_LEVELS; ++l) {
    c.channel_mult[l] = cfg->channel_mult[l]; c.num_res_blocks[l] = cfg->num_res_blocks[l];
    c.attention_resolutions[l] = cfg->attention_resolutions[l];
  }
  // every AttentionBlock's head dim must have a unet_attn instance (the output blocks' single heads included)
  Topology t = build_topology(*e);
  std::vector<Layer> all = t.middle;
  for (const std::vector<Layer>& blk : t.input_blocks) all.insert(all.end(), blk.begin(), blk.end());
  for (const std::vector<Layer>& blk : t.output_blocks) all.insert(all.end(), blk.begin(), blk.end());
  for (const Layer& L : all)
    RS_CHECK(L.kind != L_ATTN || (L.b > 0 && L.a % L.b == 0 && unet_attn_head_dim_ok(L.a / L.b)),
             "an AttentionBlock over " + std::to_string(L.a) + " channels with " + std::to_string(L.b) +
             " head(s): the attention kernel is instantiated for head dims 32, 64 and 128; set num_head_channels to "
             "32, 64 or 128 (with num_head_channels -1, output blocks have one head over all their channels)");
  int rc = build_inventory(*e); if (rc) return rc;
  *out = e.release();
  return 0;
}
int rs_unetconv_create(const rs_unetconv_config* cfg, const rs_unet_options* opts, rs_engine** out) {
  RS_CHECK(cfg && opts && out, "null argument");
  RS_CHECK(cfg->n_levels >= 1 && cfg->n_levels <= RS_MAX_LEVELS, "n_levels must be 1 .. " + std::to_string(RS_MAX_LEVELS));
  RS_CHECK(opts->patch_norm == 0, "UNetModelConv has no patch norm: rs_unet_options.patch_norm must be 0");
  for (int v : {opts->use_scale_shift_norm, opts->resblock_updown, opts->conv_resample})
    RS_CHECK(v == 0 || v == 1, "rs_unet_options fields are 0 or 1");
  RS_CHECK(cfg->dims == 2, "dims=" + std::to_string(cfg->dims) + ": only 2-D UNets are covered (set dims=2)");
  RS_CHECK(cfg->cond_lq == 1, "cond_lq must be 1: the ResShift sampler always passes lq, and the reference asserts cond_lq then");
  const int x_ch = unet_x_channels(cfg->in_channels, cfg->out_channels);
  RS_CHECK(x_ch > 0, kUnetChannelRule);
  RS_CHECK(cfg->model_channels > 0, "model_channels must be positive");
  for (int l = 0; l < cfg->n_levels; ++l) {
    RS_CHECK(cfg->channel_mult[l] > 0 && cfg->num_res_blocks[l] >= 0, "channel_mult / num_res_blocks");
    RS_CHECK(cfg->model_channels * cfg->channel_mult[l] % 8 == 0,
             "level " + std::to_string(l) + " has " + std::to_string(cfg->model_channels * cfg->channel_mult[l]) +
             " channels: the conv kernels read and write 16-byte channel rows, so model_channels * channel_mult must be a "
             "multiple of 8");
  }
  auto e = std::make_unique<rs_engine>();
  e->unetmodel = true;
  e->conv_blocks = true;
  e->opt = *opts;
  rs_unetmodel_config& u = e->um;               // the UNetModel-style input handling (x + lq, no feature extractor)
  u.in_channels = cfg->in_channels; u.out_channels = cfg->out_channels; u.model_channels = cfg->model_channels;
  u.n_levels = cfg->n_levels; u.n_attn = 0; u.num_heads = 1; u.num_head_channels = -1;
  rs_unet_config& c = e->cfg;
  std::memset(&c, 0, sizeof(c));
  c.image_size = 64; c.lq_size = 64;            // (no image_size: unused without attention levels and feature extractor)
  c.in_channels = x_ch; c.model_channels = cfg->model_channels; c.out_channels = cfg->out_channels;
  c.n_levels = cfg->n_levels; c.n_attn = 0;
  for (int l = 0; l < RS_MAX_LEVELS; ++l) {
    c.channel_mult[l] = u.channel_mult[l] = cfg->channel_mult[l];
    c.num_res_blocks[l] = u.num_res_blocks[l] = cfg->num_res_blocks[l];
  }
  int rc = build_inventory(*e); if (rc) return rc;
  *out = e.release();
  return 0;
}
void rs_unet_destroy(rs_engine* e) { delete e; }
int rs_unet_param_count(const rs_engine* e) { return e ? (int)e->params.size() : 0; }
int rs_unet_param_info(const rs_engine* e, int index, char* name, size_t name_cap, int32_t shape[4], int32_t* ndim,
                       int32_t* is_buffer) {
  RS_CHECK(e && index >= 0 && index < (int)e->params.size(), "index out of range");
  const Param& p = e->params[index];
  if (name && name_cap) { std::strncpy(name, p.name.c_str(), name_cap - 1); name[name_cap - 1] = 0; }
  for (int i = 0; i < 4; ++i) shape[i] = i < (int)p.shape.size() ? p.shape[i] : 1;
  if (ndim) *ndim = (int)p.shape.size();
  if (is_buffer) *is_buffer = (p.role == R_BUF_RELIDX || p.role == R_BUF_MASK) ? 1 : 0;
  return 0;
}
size_t rs_unet_arena_bytes(const rs_engine* e) { return e ? e->arena_bytes : 0; }
int rs_unet_set_arena(rs_engine* e, void* arena_dev) {
  RS_CHECK(e && arena_dev && (reinterpret_cast<uintptr_t>(arena_dev) & 255) == 0, "arena must be 256-byte aligned");
  int dev = -1;
  RS_CUDA_OK(cudaGetDevice(&dev));
  // the engine belongs to the current device, so device memory of another device cannot be its arena
  cudaPointerAttributes attr{};
  RS_CUDA_OK(cudaPointerGetAttributes(&attr, arena_dev));
  RS_CHECK(attr.type != cudaMemoryTypeDevice || attr.device == dev,
           "the arena is memory of cuda:" + std::to_string(attr.device) + " but cuda:" + std::to_string(dev) +
           " is current: set the arena with its device current");
  e->arena = static_cast<uint8_t*>(arena_dev);
  e->device = dev;
  return 0;
}
int rs_unet_load_param(rs_engine* e, const char* name, const float* src, void* stream) {
  RS_CHECK(e && name && src, "null argument");
  RS_CHECK(e->arena != nullptr, "rs_unet_set_arena first");
  const Param* p = e->find(name);
  RS_CHECK(p != nullptr, std::string("unknown parameter ") + name);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ++e->weights_epoch;
  if (p->bytes == 0) return 0;      // derived buffers (relative_position_index, attn_mask) are not stored
  if (p->role == R_CONV3 || p->role == R_CONV1 || p->role == R_LINEAR) {
    const int O = p->shape[0], I = p->shape[1];
    const int KH = p->shape.size() == 4 ? p->shape[2] : 1, KW = p->shape.size() == 4 ? p->shape[3] : 1;
    const long long total = (long long)O * KH * KW * p->ipad;
    (void)launch_k(pack_conv_weight_kernel, dim3((unsigned)std::min<long long>((total + 255) / 256, 4096)), dim3(256), (size_t)(0), st, 
        src, reinterpret_cast<__half*>(e->arena + p->off), O, I, KH, KW, p->ipad);
  } else if (p->role == R_RELPOS) {
    const int w = relpos_window(*p);
    RS_CHECK(w == 8 || w == 16, "relative position table must be 15x15 (window 8) or 31x31 (window 16)");
    (void)launch_k(expand_relpos_kernel, dim3((e->cfg.swin_heads * w * w * w * w + 255) / 256), dim3(256), (size_t)(0), st,
        src, reinterpret_cast<float*>(e->arena + p->off), e->cfg.swin_heads, w);
  } else {
    long long n = 1;
    for (int v : p->shape) n *= v;
    (void)launch_k(copy_f32_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), (size_t)(0), st, src, reinterpret_cast<float*>(e->arena + p->off), n);
  }
  if (!e->opt.use_scale_shift_norm) {
    // the FiLM table's bias of a ResBlock is emb_layers.1.bias + in_layers.2.bias (build_inventory); whichever of the two
    // is loaded last leaves the sum right
    const std::string nm(name);
    const char* in_bias = e->conv_blocks ? ".in_layers.1.bias" : ".in_layers.2.bias";    // (ResBlockConv: in_layers.1)
    for (const char* suffix : {".emb_layers.1.bias", in_bias}) {
      const size_t ls = std::strlen(suffix);
      if (nm.size() <= ls || nm.compare(nm.size() - ls, ls, suffix) != 0) continue;
      const std::string blk = nm.substr(0, nm.size() - ls);
      auto it = e->film_row_of.find(blk);
      if (it == e->film_row_of.end()) continue;
      const int n = p->shape[0];
      (void)launch_k(add_f32_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), (size_t)(0), st,
                     (const float*)e->at<float>(blk + ".emb_layers.1.bias"), (const float*)e->at<float>(blk + in_bias),
                     reinterpret_cast<float*>(e->arena + e->film_b_off) + it->second, n);
    }
  }
  RS_CUDA_OK(cudaGetLastError());
  return 0;
}

int rs_plan_create(rs_engine* e, int batch, int height, int width, rs_plan** out) {
  RS_CHECK(e && out && batch > 0, "bad argument");
  RS_CHECK(e->kind == EngineKind::Denoiser, std::string("this engine is ") + kind_name(e->kind) + ": use rs_vq_plan_create");
  // every level's H and W must be multiples of that level's window (the constructor-time rule: the level's nominal
  // resolution where that is not larger than window_size, else window_size)
  // (a UNetModel's levels only need to halve evenly)
  int mult = 1;
  for (int l = 0; l < e->cfg.n_levels; ++l) {
    const int res = e->cfg.image_size >> l;
    mult = e->unetmodel ? 1 << l : std::lcm(mult, (res <= e->cfg.window_size ? res : e->cfg.window_size) << l);
  }
  RS_CHECK(height % mult == 0 && width % mult == 0,
           "latent H and W must be multiples of " + std::to_string(mult) + " for this model: " +
           (e->unetmodel ? std::string("2^(levels - 1)") : std::string("each level's window (at most window_size) times the "
                                                                          "level's downsampling (64 for the shipped configs)")));
  auto p = std::make_unique<rs_plan>();
  p->e = e; p->ovr = read_overrides(); p->B = batch; p->H = height; p->W = width;
  int rc = build_plan(*p); if (rc) return rc;
  *out = p.release();
  return 0;
}
void rs_plan_destroy(rs_plan* p) { delete p; }
size_t rs_plan_workspace_bytes(const rs_plan* p) { return p ? p->workspace_bytes : 0; }
int rs_plan_num_launches(const rs_plan* p) { return p ? p->launches : 0; }

int rs_plan_bind(rs_plan* p, void* workspace_dev) {
  RS_CHECK(p && workspace_dev && (reinterpret_cast<uintptr_t>(workspace_dev) & 255) == 0, "workspace must be 256-byte aligned");
  RS_CHECK(p->e->arena != nullptr, "rs_unet_set_arena before binding a plan");
  int dev = -1;
  RS_CUDA_OK(cudaGetDevice(&dev));
  RS_CHECK(dev == p->e->device, "bind a plan on the device its engine's arena was set on (cuda:" +
                                std::to_string(p->e->device) + "), not cuda:" + std::to_string(dev));
  RS_CHECK(!p->bound || dev == p->device, "a bound plan can be rebound on its own device only");
  p->device = dev;
  p->ws = static_cast<uint8_t*>(workspace_dev);
  if (p->pass != Pass::Denoiser) {
    p->out_f32 = reinterpret_cast<float*>(p->ws + p->off_state);
  } else {
    const size_t lat = align_up((size_t)p->B * std::max(p->e->cfg.in_channels, p->e->cfg.out_channels) * p->H * p->W * 4, 256);
    p->out_f32 = reinterpret_cast<float*>(p->ws + p->off_state + lat);
  }
  resolve(*p, p->xin);
  if (p->fe_in.tens >= 0) { resolve(*p, p->fe_in); resolve(*p, p->lq_feat); }
  for (auto& kv : p->block_out) resolve(*p, kv.second);
  p->launches = 0;
  int rc = conv_init(); if (rc) return rc;
  rc = bind_ops(*p, p->fe_ops); if (rc) return rc;
  rc = bind_ops(*p, p->ops); if (rc) return rc;
  p->launches += p->pass == Pass::Denoiser ? kDenoiserOuterLaunches : p->pass == Pass::Encode ? kEncodeOuterLaunches : kDecodeOuterLaunches;
  p->bound = true;
  return 0;
}

int rs_plan_forward(rs_plan* p, const float* x, const float* timesteps, const float* lq, const float* mask, float* out,
                    void* stream) {
  RS_CHECK(p && p->bound, "plan is not bound");
  RS_CHECK(p->pass == Pass::Denoiser, std::string("this plan belongs to ") + kind_name(p->e->kind) + ": use its encode / decode calls");
  RS_CHECK(x && timesteps && lq && out, "null tensor");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = run_forward(*p, x, timesteps, lq, mask, st); if (rc) return rc;
  const long long n = (long long)p->B * p->e->cfg.out_channels * p->H * p->W;
  (void)launch_k(copy_f32_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), (size_t)(0), st, p->out_f32, out, n);
  RS_CUDA_OK(cudaGetLastError());
  return 0;
}

// One forward with a CUDA-event pair around every operator; returns time per kernel family
// (ms_by_kind[0..3] = conv/linear GEMM, GroupNorm (stats+apply), window attention, upsample) and the
// algorithmic FLOPs (2*MACs on real, un-padded channels) executed by the GEMM kernels (conv / linear, fused MLP, fused
// Swin attention) in that forward.
int rs_plan_profile(rs_plan* p, const float* x, const float* timesteps, const float* lq, const float* mask,
                    double* ms_by_kind, double* conv_flops, int32_t* n_conv_launches, void* stream) {
  RS_CHECK(p && p->bound && ms_by_kind && p->pass == Pass::Denoiser, "bad argument (needs a bound denoiser plan)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Prof prof;
  int rc = run_forward(*p, x, timesteps, lq, mask, st, &prof); if (rc) return rc;
  RS_CUDA_OK(cudaStreamSynchronize(st));
  for (int k = 0; k < 4; ++k) ms_by_kind[k] = 0.0;
  double fl = 0.0; int nc = 0;
  for (size_t i = 0; i < p->ops.size(); ++i) {
    const Op& op = p->ops[i];
    float ms = 0.f;
    cudaEventElapsedTime(&ms, prof.ev[2 * i], prof.ev[2 * i + 1]);
    int family = 0;          // GEMM kernels (FLOPs counted), GroupNorm, attention, resample
    switch (kind_of(op)) {
      case OP_CONV: {
        const ConvDesc& d = payload<ConvOp>(op).d;
        const ConvParams& c = d.prm;
        const int cin_real = d.in.tens == p->xin.tens ? p->e->cfg.in_channels + p->e->lq_feat_ch() : d.in.C;
        fl += 2.0 * (double)c.Nimg * c.Hout * c.Wout * c.Cout * (double)c.num_taps * cin_real;
        break;
      }
      case OP_MLP: { const MlpDesc& m = payload<MlpOp>(op).d; fl += 4.0 * (double)m.in.N * m.in.H * m.in.W * m.E * (double)m.Hd; break; }
      case OP_SWIN_ATTN: {   // a GEMM kernel: per token qkv 2 E 3E + proj 2 E E + (QK^T + PV over the 64 keys of its window) 4 * 64 * E
        const View& xv = payload<SwinOp>(op).d.x;
        fl += (double)xv.N * xv.H * xv.W * (8.0 * xv.C * xv.C + 256.0 * xv.C);
        break;
      }
      case OP_GN: family = 1; break;
      case OP_ATTN: case OP_SOFTMAX: case OP_VQ_ATTN: case OP_UNET_ATTN: family = 2; break;    // (no softmax / VQ-GAN attention in a denoiser)
      case OP_UPSAMPLE: family = 3; break;
    }
    ms_by_kind[family] += ms;
    nc += family == 0;
  }
  if (conv_flops) *conv_flops = fl;
  if (n_conv_launches) *n_conv_launches = nc;
  return 0;
}

// per-operator times + one-line descriptions of a profiled run_ops() pass (film_sN: the FiLM row stride it ran with)
static void collect_profile(const rs_plan& P, const Prof& prof, double* ms, char* desc, int desc_stride, int cap, int32_t* n_ops,
                            long long film_sN) {
  const int n = std::min<int>((int)P.ops.size(), cap);
  *n_ops = n;
  for (int i = 0; i < n; ++i) {
    float t = 0.f;
    cudaEventElapsedTime(&t, prof.ev[2 * i], prof.ev[2 * i + 1]);
    ms[i] = t;
    const Op& op = P.ops[i];
    char* d = desc + (size_t)i * desc_stride;
    switch (kind_of(op)) {
      case OP_CONV: {   // everything rs_op_conv2d_ex needs to replay it with the plan's epilogue, and the launch it reports
        const ConvOp& co = payload<ConvOp>(op);
        const ConvDesc& cd = co.d;
        const ConvParams& c = cd.prm;
        // the statistics sinks the kernel (or, under split-K, the reduce kernel) writes; gstat bit i: the GroupNorm that
        // reads sink i reduces its pairs with gn_finalize_kernel (many tile slots); bsN: the per-image bias row stride
        const GnSink* sk = c.splitk > 1 ? cd.red.sink : c.sink;
        const int sinks = (sk[0].part != nullptr) + (sk[1].part != nullptr);
        int gstat = 0;
        for (int k = 0; k < sinks && k < (int)co.stat_dst.size(); ++k) gstat |= gn_finalizes(co.stat_dst[k].to) ? 1 << k : 0;
        const long long bsN = co.bias_film_off >= 0 ? film_sN : 0;
        snprintf(d, desc_stride, "conv%dx%d s%d %dx%d Cin=%d Cout=%d grid=%d BN=%d st=%d %s cg=%d ms=%d sk=%d box=%dx%dx%d "
                 "N=%d persist=%d pad=%d act=%d res=%d f32=%d silu=%d film=%d bsN=%lld sinks=%d cs=%d,%d co=%d,%d gstat=%d",
                 cd.ksize, cd.ksize, cd.stride, c.Hout, c.Wout, cd.in.C, c.Cout, cd.grid, c.BN, c.stages,
                 co.w_name.c_str(), c.cg, c.msub, c.splitk, c.bw, c.bh, c.bn, c.Nimg, c.persist, cd.pad_lo,
                 cd.act, (int)cd.has_res, (int)(cd.out_f32 != nullptr), (int)cd.has_silu, (int)cd.film, bsN, sinks,
                 sk[0].cstride, sk[1].cstride, sk[0].coff, sk[1].coff, gstat);
        break;
      }
      case OP_GN: {   // everything rs_op_groupnorm_ex needs to replay it, and the launch geometry it should report
        const GnOp& o = payload<GnOp>(op);
        const GnLink& g = o.stats;
        const GnGeometry geo = gn_geometry(o.d);
        const char* route = g.win_slots ? "window_pairs" : g.fused ? (gn_finalizes(g) ? "finalize" : "conv_pairs")
                                                                   : (gn_finalizes(g) ? "stats_gstat" : "stats_pairs");
        const char* film = o.d.film_off < 0 ? "none" : film_sN > 0 ? "image" : "shared";
        snprintf(d, desc_stride, "gn %dx%d C=%d N=%d route=%s slots=%d eps=%g silu=%d film=%s@%d apply=%d rows=%d csplit=%d %s",
                 g.in.H, g.in.W, g.in.C, g.in.N, route, geo.slots, (double)g.eps, o.d.silu, film, o.d.film_off, geo.apply_ctas,
                 geo.apply_rows, geo.csplit, o.name.c_str());
        break;
      }
      case OP_MLP: { const MlpDesc& m = payload<MlpOp>(op).d; snprintf(d, desc_stride, "mlp %dx%d E=%d Hd=%d grid=%d", m.in.H, m.in.W, m.E, m.Hd, m.grid); break; }
      case OP_ATTN: {       // everything rs_op_window_attention_cfg needs to replay it, and the heads per CTA it should report
        const WinAttnOp& a = payload<WinAttnOp>(op);
        const int heads = P.e->cfg.swin_heads, hd = P.e->cfg.swin_embed_dim / heads;
        const int hpc = a.simt ? 1 : attn_default_hpc(heads, (long long)a.qkv.N * (a.qkv.H / a.window) * (a.qkv.W / a.window));
        snprintf(d, desc_stride, "attn %dx%d window=%d shift=%d N=%d heads=%d head_dim=%d hpc=%d simt=%d", a.qkv.H, a.qkv.W,
                 a.window, a.shift, a.qkv.N, heads, hd, hpc, (int)a.simt);
        break;
      }
      case OP_SWIN_ATTN: {  // ... rs_op_swin_attn_ex, with the persistent grid it should report
        const SwinAttnDesc& w = payload<SwinOp>(op).d;
        snprintf(d, desc_stride, "swin_attn %dx%d shift=%d grid=%d N=%d E=%d heads=%d slots=%d", w.x.H, w.x.W, w.shift, w.grid,
                 w.x.N, w.x.C, w.heads, w.gn_slots);
        break;
      }
      case OP_SOFTMAX: snprintf(d, desc_stride, "softmax %d", payload<SoftmaxOp>(op).view.C); break;
      case OP_VQ_ATTN: {     // the query-row range only when it is not all T rows (the default launch keeps its description)
        const VqAttnDesc& a = payload<VqAttnDesc>(op);
        if (a.row_begin == 0 && a.row_end == a.prm.T) snprintf(d, desc_stride, "vq_attn T=%d C=%d N=%d", a.prm.T, a.q.C, a.q.N);
        else snprintf(d, desc_stride, "vq_attn T=%d C=%d N=%d rows=%d:%d", a.prm.T, a.q.C, a.q.N, a.row_begin, a.row_end);
        break;
      }
      case OP_UPSAMPLE: {
        const ResampleOp& r = payload<ResampleOp>(op);
        snprintf(d, desc_stride, "%s %dx%d C=%d%s", r.pool ? "avgpool" : "upsample", r.in.H, r.in.W, r.in.C, r.has_silu ? " silu=1" : "");
        break;
      }
      case OP_UNET_ATTN: {
        const UnetAttnDesc& a = payload<UnetAttnDesc>(op);
        snprintf(d, desc_stride, "unet_attn T=%d heads=%d D=%d N=%d order=%s", a.prm.T, a.heads, a.out.C / a.heads, a.qkv.N,
                 a.new_order ? "new" : "legacy");
        break;
      }
    }
  }
}

// Per-operator timing of one forward: fills ms[i] and a short description for each op of the main program.
int rs_plan_profile_ops(rs_plan* p, const float* x, const float* timesteps, const float* lq, const float* mask,
                        double* ms, char* desc, int desc_stride, int cap, int32_t* n_ops, void* stream) {
  RS_CHECK(p && p->bound && ms && desc && n_ops, "bad argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Prof prof;
  int rc = run_forward(*p, x, timesteps, lq, mask, st, &prof); if (rc) return rc;
  RS_CUDA_OK(cudaStreamSynchronize(st));
  collect_profile(*p, prof, ms, desc, desc_stride, cap, n_ops, p->e->film_rows);
  return 0;
}

__global__ void probe_kernel(const __half* src, long long sN, int ld, float* dst, int N, int HW, int C) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * C * HW) return;
  const int hw = (int)(i % HW); const int c = (int)((i / HW) % C); const int n = (int)(i / ((long long)HW * C));
  dst[i] = __half2float(src[n * sN + (long long)hw * ld + c]);
}

int rs_plan_probe(rs_plan* p, const char* block, float* dst, int32_t* channels, int32_t* h, int32_t* w, void* stream) {
  RS_CHECK(p && p->bound && block, "bad argument");
  if (dst) { int rc = check_plan_device(*p); if (rc) return rc; }
  auto it = p->block_out.find(block);
  RS_CHECK(it != p->block_out.end(), std::string("unknown block ") + block);
  const View& v = it->second;
  if (channels) *channels = v.C; if (h) *h = v.H; if (w) *w = v.W;
  if (dst) {
    const long long n = (long long)v.N * v.C * v.H * v.W;
    (void)launch_k(probe_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), (size_t)(0), static_cast<cudaStream_t>(stream), v.ptr, v.sN(), v.ld, dst, v.N, v.H * v.W, v.C);
    RS_CUDA_OK(cudaGetLastError());
  }
  return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// sampler
// ------------------------------------------------------------------------------------------------
struct rs_sampler {
  rs_plan* p = nullptr;
  int T = 0;
  // the process (StepProcess) and the scalars its step reads
  int process = kStepResShift;
  int mean_type = RS_MEAN_XSTART;
  int clip = 0;                 // DDPM processes: clamp x0 to [-1, 1]
  float eta = 0;                // DDIM
  float prior_coef = 0;         // ResShift: kappa * sqrt_eta[T - 1]
  int var_mode = 0;             // StepVar of the ancestral step (kVarFixed for every other process)
  // rows x T fp32: row r is what the plan's table region holds at r * 1024 (the process's row enum)
  int rows = 0;
  std::vector<float> tab;
  std::vector<float> tsteps;    // [T] the model's timesteps
  float* tap_pred = nullptr; float* tap_sample = nullptr;
  cudaGraphExec_t graph = nullptr;
  cudaStream_t cap_stream = nullptr;     // capture happens on a private stream (the legacy default stream cannot capture)
  const void* g_zy = nullptr; const void* g_noise = nullptr; const void* g_lq = nullptr; const void* g_mask = nullptr;
  void* g_out = nullptr;
};

namespace {

static_assert((int)kMeanXstart == (int)RS_MEAN_XSTART && (int)kMeanEpsilon == (int)RS_MEAN_EPSILON &&
              (int)kMeanEpsilonScale == (int)RS_MEAN_EPSILON_SCALE && (int)kMeanResidual == (int)RS_MEAN_RESIDUAL,
              "MeanType mirrors rs_mean_type");
static_assert(kRsRows <= kStepRows && kDdRows <= kStepRows && kInvRows <= kStepRows, "the table region holds every row");

// what rs_sampler_run reads of a process: z_y (the ResShift conditioning, or the inversion's x_start), and the T + 1
// noises (the first state, then one per step) of every process but inversion
bool reads_zy(const rs_sampler& s) { return s.process == kStepResShift || s.process == kStepInversion; }
size_t noise_count(const rs_sampler& s) { return s.process == kStepInversion ? 0 : (size_t)s.T + 1; }
// whether the step at t has a next step (whose denoiser input it packs): t walks down to 0, or up to T - 1 in inversion
bool step_has_next(int process, int t, int T) { return process == kStepInversion ? t + 1 < T : t > 0; }

// the step_kernel instance of (process, mean type, output layout), with the grid every caller launches; combinations
// without an instance are refused.  A packed output (out_sN = C * HW) runs the fixed instances; the ancestral step's
// learned modes, and DDIM / inversion on a wider stride, run the strided ones.  The ResShift xstart instance writes no
// x0: x0_out receives a copy of the model output, ahead.
int launch_step(int process, int mean_type, const StepParams& sp, cudaStream_t st) {
  const long long numel = (long long)sp.N * sp.C * sp.HW;
  const dim3 grid((unsigned)((numel + 255) / 256)), block(256);
  auto go = [&](void (*kernel)(const StepParams)) {
    (void)launch_k(kernel, grid, block, (size_t)(0), st, sp);
    RS_CUDA_OK(cudaGetLastError());
    return 0;
  };
  const bool eps = mean_type == RS_MEAN_EPSILON, x0 = mean_type == RS_MEAN_XSTART;
  const bool packed = sp.out_sN == (long long)sp.C * sp.HW, learned = sp.var_mode != kVarFixed;
  RS_CHECK(sp.out_sN >= (long long)sp.C * sp.HW * (learned ? 2 : 1) && (process == kStepAncestral || !learned) &&
           (packed || learned || process == kStepDdim || process == kStepInversion),
           "step: no layout for var mode " + std::to_string(sp.var_mode) + " at image stride " + std::to_string(sp.out_sN));
  switch (process) {
    case kStepResShift:
      if (x0 && sp.x0_out) RS_CUDA_OK(cudaMemcpyAsync(sp.x0_out, sp.out, (size_t)numel * 4, cudaMemcpyDeviceToDevice, st));
      if (x0) return go(step_kernel<kStepResShift, kMeanXstart>);
      if (eps) return go(step_kernel<kStepResShift, kMeanEpsilon>);
      if (mean_type == RS_MEAN_EPSILON_SCALE) return go(step_kernel<kStepResShift, kMeanEpsilonScale>);
      if (mean_type == RS_MEAN_RESIDUAL) return go(step_kernel<kStepResShift, kMeanResidual>);
      break;
    case kStepAncestral:
      if (sp.var_mode == kVarLearned) {
        if (eps) return go(step_kernel<kStepAncestral, kMeanEpsilon, kVarLearned>);
        if (x0) return go(step_kernel<kStepAncestral, kMeanXstart, kVarLearned>);
      } else if (sp.var_mode == kVarLearnedRange) {
        if (eps) return go(step_kernel<kStepAncestral, kMeanEpsilon, kVarLearnedRange>);
        if (x0) return go(step_kernel<kStepAncestral, kMeanXstart, kVarLearnedRange>);
      } else {
        if (eps) return go(step_kernel<kStepAncestral, kMeanEpsilon>);
        if (x0) return go(step_kernel<kStepAncestral, kMeanXstart>);
      }
      break;
    case kStepDdim:
      if (eps) return go(packed ? step_kernel<kStepDdim, kMeanEpsilon> : step_kernel<kStepDdim, kMeanEpsilon, kVarLearned>);
      if (x0) return go(packed ? step_kernel<kStepDdim, kMeanXstart> : step_kernel<kStepDdim, kMeanXstart, kVarLearned>);
      break;
    case kStepInversion:
      if (eps) return go(packed ? step_kernel<kStepInversion, kMeanEpsilon> : step_kernel<kStepInversion, kMeanEpsilon, kVarLearned>);
      if (x0) return go(packed ? step_kernel<kStepInversion, kMeanXstart> : step_kernel<kStepInversion, kMeanXstart, kVarLearned>);
      break;
  }
  return ::rs::fail(-1, "no step kernel for process " + std::to_string(process) + " and mean type " + std::to_string(mean_type));
}

// The fused loop of every process.  x at the first step is x_T = z_y + kappa sqrt_eta_T noises[0] (ResShift
// prior_sample), noises[0] (ancestral, DDIM) or z_y (inversion's x_start); then per step the denoiser on x (scaled by
// in_scale[t] for ResShift) with FiLM row t, and one step launch; the last step writes out_latent.
int sampler_enqueue(rs_sampler& S, const float* z_y, const float* noises, const float* lq, const float* mask,
                    float* out_latent, cudaStream_t st) {
  rs_plan& P = *S.p;
  const rs_unet_config& c = P.e->cfg;
  // the DDPM processes' output width was checked against the variance type when the sampler was made
  RS_CHECK(S.process != kStepResShift || c.in_channels == c.out_channels,
           "the sampler needs out_channels == in_channels (x0 and x_t share a shape)");
  const long long numel = (long long)P.B * c.in_channels * P.H * P.W;
  float* state = reinterpret_cast<float*>(P.ws + P.off_state);
  const float* tab = reinterpret_cast<const float*>(P.ws + P.off_tables);
  const bool resshift = S.process == kStepResShift, inversion = S.process == kStepInversion;
  const float* x = inversion ? z_y : noises;
  if (resshift) {
    (void)launch_k(prior_sample_kernel, dim3((unsigned)((numel + 255) / 256)), dim3(256), (size_t)(0), st, z_y, noises, state, S.prior_coef, numel);
    x = state;
  }
  // LQ feature (once) + the first packed input
  int rc = pack_lq_and_input(P, x, lq, mask, resshift ? tab + kRsInScale * 1024 : nullptr, S.T - 1, st); if (rc) return rc;
  const float* film_all = reinterpret_cast<const float*>(P.ws + P.off_film);
  StepParams sp{};
  sp.out = P.out_f32; sp.y = z_y;
  for (int r = 0; r < S.rows; ++r) sp.row[r] = tab + r * 1024;
  sp.eta = S.eta; sp.clip = S.clip;
  sp.N = P.B; sp.C = c.in_channels; sp.HW = P.H * P.W;
  sp.out_sN = (long long)c.out_channels * sp.HW; sp.var_mode = S.var_mode;
  sp.next_cpad = P.cin_pad;
  sp.zero_ptr = reinterpret_cast<unsigned int*>(P.ws + P.off_counters); sp.zero_n = P.n_gn * P.B;
  for (int k = 0; k < S.T; ++k) {
    const int t = inversion ? k : S.T - 1 - k;
    rc = run_ops(P, P.ops, film_all + (long long)t * P.e->film_rows, 0, st); if (rc) return rc;
    sp.x_t = k == 0 ? x : state;
    sp.noise = inversion ? nullptr : noises + (long long)(k + 1) * numel;
    sp.x_next = k == S.T - 1 ? out_latent : state;
    sp.t = t;
    sp.next_in = step_has_next(S.process, t, S.T) ? P.xin.ptr : nullptr;
    sp.x0_out = S.tap_pred ? S.tap_pred + (long long)k * numel : nullptr;
    rc = launch_step(S.process, S.mean_type, sp, st); if (rc) return rc;
    if (S.tap_sample) RS_CUDA_OK(cudaMemcpyAsync(S.tap_sample + (long long)k * numel, sp.x_next, numel * 4, cudaMemcpyDeviceToDevice, st));
  }
  RS_CUDA_OK(cudaGetLastError());
  return 0;
}

int sampler_prepare(rs_sampler& S, cudaStream_t st) {
  // tables + the FiLM table of all T steps (depends on the timestep only: reference models/unet.py:874,
  // models/respace.py:60-63) — computed once, outside any graph capture.
  rs_plan& P = *S.p;
  if (P.table_owner == &S && P.table_epoch == P.e->weights_epoch) return 0;
  float* tab = reinterpret_cast<float*>(P.ws + P.off_tables);
  for (int r = 0; r < S.rows; ++r)
    RS_CUDA_OK(cudaMemcpyAsync(tab + r * 1024, S.tab.data() + (size_t)r * S.T, S.T * 4, cudaMemcpyHostToDevice, st));
  float* ts = reinterpret_cast<float*>(P.ws + P.off_tsteps);
  RS_CUDA_OK(cudaMemcpyAsync(ts, S.tsteps.data(), S.T * 4, cudaMemcpyHostToDevice, st));
  int rc = run_embedding(P, ts, S.T, st); if (rc) return rc;
  RS_CUDA_OK(cudaStreamSynchronize(st));     // host vectors must outlive the copies; one-time setup cost
  P.table_owner = &S; P.table_epoch = P.e->weights_epoch;
  return 0;
}

}  // namespace

extern "C" {

// posterior tables in float64, cast to fp32 like _extract_into_tensor (reference models/gaussian_diffusion.py:92-105,143-161)
// in_scale follows _scale_input (:598-609): 1 / sqrt(eta kappa^2 + 1) with latent_flag, 1 / (sqrt_eta kappa 3 + 1)
// without, 1 without normalize_input; every operation of the reference's fp32 expression rounded in fp32 on its fp32
// table value.  eps_coef, eta and one_minus_eta are the fp32 factors of _predict_xstart_from_eps / _eps_scale (:308-318).
static void schedule_tables(rs_sampler& s, int steps, const double* sqrt_etas, double kappa, const int32_t* tmap,
                            const rs_sampler_options& opt = rs_sampler_options{RS_MEAN_XSTART, 1, 1}) {
  std::vector<double> etas(steps), prev(steps), alpha(steps), pv(steps);
  for (int i = 0; i < steps; ++i) etas[i] = sqrt_etas[i] * sqrt_etas[i];
  for (int i = 0; i < steps; ++i) { prev[i] = i ? etas[i - 1] : 0.0; alpha[i] = etas[i] - prev[i]; pv[i] = kappa * kappa * prev[i] / etas[i] * alpha[i]; }
  s.T = steps; s.rows = kRsRows; s.mean_type = opt.mean_type;
  s.tab.resize((size_t)kRsRows * steps); s.tsteps.resize(steps);
  float* row[kRsRows];
  for (int r = 0; r < kRsRows; ++r) row[r] = s.tab.data() + (size_t)r * steps;
  for (int i = 0; i < steps; ++i) {
    const double pvc = pv[i == 0 ? 1 : i];
    row[kRsCoef1][i] = (float)(prev[i] / etas[i]);
    row[kRsCoef2][i] = (float)(alpha[i] / etas[i]);
    const float logv = (float)std::log(pvc);
    row[kRsStd][i] = std::exp(0.5f * logv);
    const float e32 = (float)etas[i];
    if (!opt.normalize_input) {
      row[kRsInScale][i] = 1.0f;
    } else if (opt.latent_flag) {
      row[kRsInScale][i] = 1.0f / std::sqrt(e32 * (float)(kappa * kappa) + 1.0f);
    } else {
      row[kRsInScale][i] = 1.0f / ((float)sqrt_etas[i] * (float)kappa * 3.0f + 1.0f);
    }
    s.tsteps[i] = (float)(tmap ? tmap[i] : i);
    row[kRsEpsCoef][i] = (float)sqrt_etas[i] * (float)kappa;
    row[kRsEta][i] = e32;
    row[kRsOneMinusEta][i] = (float)(1.0 - etas[i]);
  }
  s.prior_coef = (float)(kappa * sqrt_etas[steps - 1]);
}

static int check_sampler_options(const rs_sampler_options& o) {
  RS_CHECK(o.mean_type >= RS_MEAN_XSTART && o.mean_type <= RS_MEAN_RESIDUAL,
           "unknown mean type " + std::to_string(o.mean_type) + " (RS_MEAN_XSTART .. RS_MEAN_RESIDUAL)");
  RS_CHECK((o.normalize_input == 0 || o.normalize_input == 1) && (o.latent_flag == 0 || o.latent_flag == 1),
           "normalize_input and latent_flag must be 0 or 1");
  return 0;
}

// rs_sampler_tables' layout: coef1, coef2, std, in_scale, the timesteps (T each), then the prior coefficient; returns
// the end of what it wrote
static float* copy_tables(const rs_sampler& s, float* dst) {
  std::memcpy(dst, s.tab.data(), (size_t)4 * s.T * sizeof(float));
  std::memcpy(dst + 4 * s.T, s.tsteps.data(), (size_t)s.T * sizeof(float));
  dst[5 * s.T] = s.prior_coef;
  return dst + 5 * s.T + 1;
}

// A sampler of `process` on plan p (bound): the checks every sampler shares (`who` names it in the steps refusal),
// the timestep row, and table row r = the float64 row rows[r] of `tables` ([*][steps], rs_ddpm_table_row order)
// rounded to fp32 as _extract_into_tensor does (reference models/gaussian_diffusion.py:92-105)
static int sampler_new(rs_plan* p, int process, int steps, const int32_t* tmap, const char* who, const double* tables,
                       std::initializer_list<int> rows, std::unique_ptr<rs_sampler>& s) {
  RS_CHECK(p->pass == Pass::Denoiser, std::string("samplers are built on denoiser plans: this plan belongs to ") + kind_name(p->e->kind));
  RS_CHECK(steps >= 2 && steps <= p->max_rows && steps <= 1024,
           std::string(who) + ": steps must be in [2, " + std::to_string(std::min(p->max_rows, 1024)) +
           "] (the plan's FiLM-table rows), got " + std::to_string(steps));
  s = std::make_unique<rs_sampler>();
  s->p = p; s->process = process; s->T = steps; s->rows = (int)rows.size();
  s->tab.resize(rows.size() * steps);
  float* dst = s->tab.data();
  for (int r : rows)
    for (int i = 0; i < steps; ++i) *dst++ = (float)tables[(size_t)r * steps + i];
  s->tsteps.resize(steps);
  for (int i = 0; i < steps; ++i) s->tsteps[i] = (float)(tmap ? tmap[i] : i);
  return 0;
}

int rs_sampler_create_ex(rs_plan* p, int steps, const double* sqrt_etas, double kappa, const int32_t* tmap,
                         const rs_sampler_options* opt, rs_sampler** out) {
  RS_CHECK(p && p->bound && sqrt_etas && opt && out, "bad argument (plan must be bound)");
  int rc = check_sampler_options(*opt); if (rc) return rc;
  std::unique_ptr<rs_sampler> s;
  rc = sampler_new(p, kStepResShift, steps, tmap, "ResShift sampler", nullptr, {}, s); if (rc) return rc;
  schedule_tables(*s, steps, sqrt_etas, kappa, tmap, *opt);
  *out = s.release();
  return 0;
}
int rs_sampler_create(rs_plan* p, int steps, const double* sqrt_etas, double kappa, const int32_t* tmap, rs_sampler** out) {
  const rs_sampler_options opt{RS_MEAN_XSTART, 1, 1};
  return rs_sampler_create_ex(p, steps, sqrt_etas, kappa, tmap, &opt, out);
}
// DDPM / DDIM sampler: the process's float64 tables (rs_ddpm_table_row) rounded to fp32 as _extract_into_tensor does
// (reference models/gaussian_diffusion.py:92-105); the log-variance row of the options' var_type (:788-801)
int rs_ddpm_sampler_create(rs_plan* p, int steps, const double* tables, const int32_t* tmap, const rs_ddpm_options* o,
                           rs_sampler** out) {
  RS_CHECK(p && p->bound && out, "bad argument (plan must be bound)");
  RS_CHECK(tables, "DDPM sampler: the schedule tables are NULL");
  RS_CHECK(o, "DDPM sampler: the options are NULL");
  RS_CHECK(o->kind == RS_DDPM_ANCESTRAL || o->kind == RS_DDPM_DDIM,
           "DDPM sampler: unknown kind " + std::to_string(o->kind) + " (RS_DDPM_ANCESTRAL or RS_DDPM_DDIM)");
  RS_CHECK(o->mean_type == RS_MEAN_EPSILON || o->mean_type == RS_MEAN_XSTART,
           "DDPM sampler: the model must predict eps or x0 (RS_MEAN_EPSILON or RS_MEAN_XSTART), got mean type " +
           std::to_string(o->mean_type));
  const bool learned = o->var_type == RS_VAR_LEARNED || o->var_type == RS_VAR_LEARNED_RANGE;
  RS_CHECK(o->var_type == RS_VAR_FIXED_LARGE || o->var_type == RS_VAR_FIXED_SMALL || learned,
           "DDPM sampler: unknown variance type " + std::to_string(o->var_type) +
           " (RS_VAR_FIXED_LARGE, RS_VAR_FIXED_SMALL, RS_VAR_LEARNED_RANGE or RS_VAR_LEARNED)");
  RS_CHECK(o->clip == 0 || o->clip == 1, "DDPM sampler: clip must be 0 or 1, got " + std::to_string(o->clip));
  RS_CHECK(std::isfinite(o->eta) && o->eta >= 0.0, "DDPM sampler: eta must be finite and >= 0, got " + std::to_string(o->eta));
  // the model output: the mean (C channels, as x), then with a learned variance the variance values (C more)
  const rs_unet_config& c = p->e->cfg;
  RS_CHECK(c.out_channels == c.in_channels * (learned ? 2 : 1),
           std::string("DDPM sampler: ") + (learned ? "a learned" : "a fixed") + " variance type (" +
           std::to_string(o->var_type) + ") needs a model with " + std::to_string(c.in_channels * (learned ? 2 : 1)) +
           " output channels (" + (learned ? "twice" : "as many as") + " the " + std::to_string(c.in_channels) +
           " channels of x), this plan's model has " + std::to_string(c.out_channels));
  std::unique_ptr<rs_sampler> s;
  static_assert(kDdSqrtRecipAcp == 0 && kDdSqrtRecipm1Acp == 1 && kDdCoef1 == 2 && kDdCoef2 == 3 && kDdLogVar == 4 &&
                kDdAcp == 5 && kDdAcpPrev == 6 && kDdLogBetas == 7, "the rows below are in DdpmRow order");
  const int logvar_row = o->var_type == RS_VAR_FIXED_LARGE ? RS_DDPM_LOGVAR_LARGE : RS_DDPM_LOGVAR_SMALL;
  const int process = o->kind == RS_DDPM_DDIM ? kStepDdim : kStepAncestral;
  int rc = o->var_type == RS_VAR_LEARNED_RANGE
               ? sampler_new(p, process, steps, tmap, "DDPM sampler", tables,
                             {RS_DDPM_SQRT_RECIP_ACP, RS_DDPM_SQRT_RECIPM1_ACP, RS_DDPM_COEF1, RS_DDPM_COEF2, logvar_row,
                              RS_DDPM_ACP, RS_DDPM_ACP_PREV, RS_DDPM_LOG_BETAS}, s)
               : sampler_new(p, process, steps, tmap, "DDPM sampler", tables,
                             {RS_DDPM_SQRT_RECIP_ACP, RS_DDPM_SQRT_RECIPM1_ACP, RS_DDPM_COEF1, RS_DDPM_COEF2, logvar_row,
                              RS_DDPM_ACP, RS_DDPM_ACP_PREV}, s);
  if (rc) return rc;
  s->mean_type = o->mean_type; s->clip = o->clip; s->eta = (float)o->eta;
  if (process == kStepAncestral && learned) s->var_mode = o->var_type == RS_VAR_LEARNED ? kVarLearned : kVarLearnedRange;
  *out = s.release();
  return 0;
}
// DDIM inversion sampler: sqrt_recip_acp, sqrt_recipm1_acp and acp_next of the process's float64 tables, rounded to
// fp32 as _extract_into_tensor does (reference models/gaussian_diffusion.py:92-105, :1054-1058)
int rs_ddim_reverse_sampler_create(rs_plan* p, int steps, const double* tables, const int32_t* tmap,
                                   const rs_ddim_reverse_options* o, rs_sampler** out) {
  RS_CHECK(p && p->bound && out, "bad argument (plan must be bound)");
  RS_CHECK(tables, "DDIM reverse sampler: the schedule tables are NULL");
  RS_CHECK(o, "DDIM reverse sampler: the options are NULL");
  RS_CHECK(o->mean_type == RS_MEAN_EPSILON || o->mean_type == RS_MEAN_XSTART,
           "DDIM reverse sampler: the model must predict eps or x0 (RS_MEAN_EPSILON or RS_MEAN_XSTART), got mean type " +
           std::to_string(o->mean_type));
  RS_CHECK(o->clip == 0 || o->clip == 1, "DDIM reverse sampler: clip must be 0 or 1, got " + std::to_string(o->clip));
  const rs_unet_config& c = p->e->cfg;
  RS_CHECK(c.out_channels == c.in_channels || c.out_channels == 2 * c.in_channels,
           "DDIM reverse sampler: the model must output as many channels as x has (" + std::to_string(c.in_channels) +
           ") or twice as many (a learned variance), this plan's model has " + std::to_string(c.out_channels));
  std::unique_ptr<rs_sampler> s;
  static_assert(kInvSqrtRecipAcp == 0 && kInvSqrtRecipm1Acp == 1 && kInvAcpNext == 2, "the rows below are in InversionRow order");
  int rc = sampler_new(p, kStepInversion, steps, tmap, "DDIM reverse sampler", tables,
                       {RS_DDPM_SQRT_RECIP_ACP, RS_DDPM_SQRT_RECIPM1_ACP, RS_DDPM_ACP_NEXT}, s);
  if (rc) return rc;
  s->mean_type = o->mean_type; s->clip = o->clip;
  *out = s.release();
  return 0;
}
int rs_sampler_tables(const rs_sampler* s, float* dst) {
  RS_CHECK(s && dst, "null argument");
  RS_CHECK(s->process == kStepResShift, "rs_sampler_tables: a DDPM sampler has no residual-shift tables");
  copy_tables(*s, dst);
  return 0;
}
int rs_plan_embedding(rs_plan* p, const float* tsteps, int rows, float* sin_out, float* mid_out, float* vec_out,
                      float* film_out, void* stream) {
  RS_CHECK(p && p->bound && tsteps, "bad argument (plan must be bound)");
  RS_CHECK(p->pass == Pass::Denoiser, std::string("not a denoiser plan: this plan belongs to ") + kind_name(p->e->kind));
  RS_CHECK(rows >= 1 && rows <= p->max_rows, "rows must be in [1, " + std::to_string(p->max_rows) + "], got " + std::to_string(rows));
  int rc = check_plan_device(*p); if (rc) return rc;
  rs_plan& P = *p;
  const rs_engine& E = *P.e;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  P.table_owner = nullptr;                       // the FiLM rows a sampler keeps are overwritten
  rc = run_embedding(P, tsteps, rows, st); if (rc) return rc;
  const size_t K = (size_t)E.time_dim();
  const struct { float* dst; size_t off, width; } outs[4] = {
      {sin_out, P.off_emb_sin, (size_t)E.cfg.model_channels}, {mid_out, P.off_emb_mid, K}, {vec_out, P.off_emb_vec, K},
      {film_out, P.off_film, (size_t)E.film_rows}};
  for (const auto& o : outs)
    if (o.dst) RS_CUDA_OK(cudaMemcpyAsync(o.dst, P.ws + o.off, (size_t)rows * o.width * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}
int rs_schedule_tables(int steps, const double* sqrt_etas, double kappa, const int32_t* tmap, float* dst) {
  RS_CHECK(sqrt_etas && dst && steps >= 1, "bad argument");
  rs_sampler s;
  schedule_tables(s, steps, sqrt_etas, kappa, tmap);
  copy_tables(s, dst);
  return 0;
}
int rs_schedule_tables_ex(int steps, const double* sqrt_etas, double kappa, const int32_t* tmap,
                          const rs_sampler_options* opt, float* dst) {
  RS_CHECK(sqrt_etas && opt && dst && steps >= 1, "bad argument");
  int rc = check_sampler_options(*opt); if (rc) return rc;
  rs_sampler s;
  schedule_tables(s, steps, sqrt_etas, kappa, tmap, *opt);
  dst = copy_tables(s, dst);
  std::memcpy(dst, s.tab.data() + (size_t)kRsEpsCoef * steps, (size_t)3 * steps * sizeof(float));   // eps_coef, eta, 1 - eta
  return 0;
}
void rs_sampler_destroy(rs_sampler* s) {
  if (s && s->p && s->p->table_owner == s) s->p->table_owner = nullptr;
  if (s && s->graph) cudaGraphExecDestroy(s->graph);
  if (s && s->cap_stream) cudaStreamDestroy(s->cap_stream);
  delete s;
}
int rs_sampler_set_taps(rs_sampler* s, float* pred, float* sample) {
  RS_CHECK(s, "null sampler");
  s->tap_pred = pred; s->tap_sample = sample;
  if (s->graph) { cudaGraphExecDestroy(s->graph); s->graph = nullptr; }
  return 0;
}

int rs_sampler_run(rs_sampler* s, const float* z_y, const float* noises, const float* lq, const float* mask,
                   float* out_latent, int use_graph, void* stream) {
  RS_CHECK(!(s && s->process == kStepInversion) || z_y, "DDIM reverse sampler: x_start (z_y) is NULL");
  RS_CHECK(s && (z_y || !reads_zy(*s)) && (noises || !noise_count(*s)) && lq && out_latent, "null argument");
  int rc = check_plan_device(*s->p); if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  rc = sampler_prepare(*s, st); if (rc) return rc;
  if (!use_graph) return sampler_enqueue(*s, z_y, noises, lq, mask, out_latent, st);
  if (s->graph && (s->g_zy != z_y || s->g_noise != noises || s->g_lq != lq || s->g_mask != mask || s->g_out != out_latent)) {
    cudaGraphExecDestroy(s->graph); s->graph = nullptr;
  }
  if (!s->graph) {
    cudaGraph_t g = nullptr;
    if (!s->cap_stream) RS_CUDA_OK(cudaStreamCreateWithFlags(&s->cap_stream, cudaStreamNonBlocking));
    RS_CUDA_OK(cudaStreamBeginCapture(s->cap_stream, cudaStreamCaptureModeThreadLocal));
    rc = sampler_enqueue(*s, z_y, noises, lq, mask, out_latent, s->cap_stream);
    cudaError_t ce = cudaStreamEndCapture(s->cap_stream, &g);
    if (rc) { if (g) cudaGraphDestroy(g); return rc; }
    RS_CUDA_OK(ce);
    RS_CUDA_OK(cudaGraphInstantiate(&s->graph, g, 0));
    cudaGraphDestroy(g);
    s->g_zy = z_y; s->g_noise = noises; s->g_lq = lq; s->g_mask = mask; s->g_out = out_latent;
  }
  RS_CUDA_OK(cudaGraphLaunch(s->graph, st));
  return 0;
}

size_t rs_sampler_staging_bytes(const rs_sampler* s) {
  if (!s) return 0;
  const rs_plan& P = *s->p;
  const rs_unet_config& c = P.e->cfg;
  const size_t lat = align_up((size_t)P.B * c.in_channels * P.H * P.W * 4, 256);
  const size_t lq = align_up((size_t)P.B * 3 * P.lqH * P.lqW * 4, 256);
  const size_t mk = align_up((size_t)P.B * 1 * P.lqH * P.lqW * 4, 256);
  return lat * (noise_count(*s) + 2) + lq + mk;
}

int rs_sampler_run_host(rs_sampler* s, const float* z_y_h, const float* noises_h, const float* lq_h, const float* mask_h,
                        float* out_h, void* staging, size_t staging_bytes, int use_graph, void* stream) {
  RS_CHECK(!(s && s->process == kStepInversion) || z_y_h, "DDIM reverse sampler: x_start (z_y) is NULL");
  RS_CHECK(s && (z_y_h || !reads_zy(*s)) && (noises_h || !noise_count(*s)) && lq_h && out_h && staging, "null argument");
  RS_CHECK(staging_bytes >= rs_sampler_staging_bytes(s), "staging buffer too small");
  { int rc = check_plan_device(*s->p); if (rc) return rc; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const rs_plan& P = *s->p;
  const rs_unet_config& c = P.e->cfg;
  const size_t n_lat = (size_t)P.B * c.in_channels * P.H * P.W;
  const size_t lat = align_up(n_lat * 4, 256);
  const size_t n_lq = (size_t)P.B * 3 * P.lqH * P.lqW, n_mk = (size_t)P.B * P.lqH * P.lqW;
  uint8_t* base = static_cast<uint8_t*>(staging);
  float* d_zy = reinterpret_cast<float*>(base);
  float* d_out = reinterpret_cast<float*>(base + lat);
  const size_t n_noise = noise_count(*s);
  float* d_noise = reinterpret_cast<float*>(base + 2 * lat);
  float* d_lq = reinterpret_cast<float*>(base + lat * (n_noise + 2));
  float* d_mask = reinterpret_cast<float*>(base + lat * (n_noise + 2) + align_up(n_lq * 4, 256));
  if (z_y_h) RS_CUDA_OK(cudaMemcpyAsync(d_zy, z_y_h, n_lat * 4, cudaMemcpyHostToDevice, st));
  if (n_noise) RS_CUDA_OK(cudaMemcpyAsync(d_noise, noises_h, n_lat * 4 * n_noise, cudaMemcpyHostToDevice, st));
  RS_CUDA_OK(cudaMemcpyAsync(d_lq, lq_h, n_lq * 4, cudaMemcpyHostToDevice, st));
  if (mask_h) RS_CUDA_OK(cudaMemcpyAsync(d_mask, mask_h, n_mk * 4, cudaMemcpyHostToDevice, st));
  int rc = rs_sampler_run(s, z_y_h ? d_zy : nullptr, n_noise ? d_noise : nullptr, d_lq, mask_h ? d_mask : nullptr, d_out,
                          use_graph, stream);
  if (rc) return rc;
  RS_CUDA_OK(cudaMemcpyAsync(out_h, d_out, n_lat * 4, cudaMemcpyDeviceToHost, st));
  RS_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

__global__ void p_sample_flat_kernel(const float* x, const float* x0, const float* nz, float* out, float c1, float c2,
                                     float sd, int t0, long long n) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v = c1 * x[i] + c2 * x0[i];
  if (!t0) v += sd * nz[i];
  out[i] = v;
}
int rs_p_sample(const float* x_t, const float* x0, const float* noise, float* x_next, float c1, float c2, float sd,
                int t_is_zero, long long numel, void* stream) {
  RS_CHECK(x_t && x0 && noise && x_next && numel > 0, "bad argument");
  (void)launch_k(p_sample_flat_kernel, dim3((unsigned)((numel + 255) / 256)), dim3(256), (size_t)(0), static_cast<cudaStream_t>(stream), 
      x_t, x0, noise, x_next, c1, c2, sd, t_is_zero, numel);
  RS_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // extern "C"

#include "vq.inc"
#include "ops_api.inc"
