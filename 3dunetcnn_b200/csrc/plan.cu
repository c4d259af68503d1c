// Whole-network executor: builds, once per (architecture, input shape), the static schedule of kernels that
// reproduces the reference UNet3D forward and its autograd backward, over a caller-provided workspace arena.
//
// Reference graph restated (paths relative to /root/reference):
//   encoder      unet3d/models/pytorch/segmentation/unet.py:7-16 + classification/myronenko.py:83-107
//   res. block   classification/myronenko.py:34-58  (GN -> ReLU -> conv) x2 + identity / 1x1x1 `sample`
//   decoder      segmentation/unet.py:19-44 + classification/decoder.py:73-130 (1x1x1 pre-conv, trilinear x2, concat)
//   head         autoencoder/variational.py:59-60,81-87
// State-dict order/shapes follow SURVEY.md appendix B so reference checkpoints bind by position.
#include <functional>
#include <string>
#include <vector>
#include <cstring>
#include <cstdio>
#include <cstdlib>

#include "kernels.h"
#include "../../include/b200unet.h"

namespace b200 {

struct ParamInfo {
  std::string key;
  int64_t shape[5];
  int ndim;
};

struct Buf {
  size_t off_hi, off_lo;
  int N, D, H, W, C;
  long long stats_off;  // offset (bytes) of [N][C][2] doubles in the stats arena, or -1
};

struct TRef {
  int buf;
  int c0, c;
  int vis_m1;   // 1: the last plane/row/column is masked (reads as zero through TMA): dU of a padded ConvTranspose3d
  bool valid() const { return buf >= 0; }
};
static const TRef kNone = {-1, 0, 0, 0};

struct RunCtx {
  uint8_t* ws;                     // the caller's workspace, aligned up to 1 KiB
  const float* const* params = nullptr;
  float* const* grads = nullptr;
  const float* x = nullptr;
  float* logits = nullptr;
  const float* dlogits = nullptr;
  const float* drop = nullptr;
  float* dx = nullptr;             // input-gradient ops only: NCDHW fp32 gradient of the network input
  cudaStream_t st;
  int launches = 0;
  struct Prof* prof;
  const char* label = nullptr;     // name of the op being launched (profiling only)
  bool skip_pack = false;          // the packed bf16 weights in the workspace are current (parameters unchanged since the last forward)
  RunCtx(void* workspace, void* stream, struct Prof* p)
      : ws(reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(workspace) + 1023) & ~uintptr_t(1023))),
        st(reinterpret_cast<cudaStream_t>(stream)), prof(p) {}
};

// launch categories of the per-kernel profile (models.py _Plan.CATEGORIES names them in this order)
enum Cat { CAT_CONV_FWD = 0, CAT_CONV_DGRAD, CAT_CONV_WGRAD, CAT_NORM, CAT_RESAMPLE, CAT_HEAD, CAT_PACK, CAT_OTHER, CAT_COUNT };

struct Prof {
  std::vector<cudaEvent_t> ev;    // 2 per launch
  std::vector<int> cat;
  std::vector<std::string> label;
  size_t used = 0;                // launches recorded
  bool overflow = false;
};

enum LayerKind {
  LAYER_CONV = 0,          // nn.Conv3d, weight [Co][Ci][T], padding ksz / 2
  LAYER_CONVT_ZI,          // nn.ConvTranspose3d(k3, s2, p1) + bias parameter pb, weight [Ci][Co][T]: run as a stride-1 conv over
                           // the zero-inserted input (ksz 3, stride 1), the high boundary of its output forced to 0
  LAYER_CONVT_K2S2,        // ConvTranspose3d with kernel = stride = 2 (MONAI UnetUpBlock): ksz 2, stride 2, weight [Ci][Co][8], no padding
};
enum ConvDir { DIR_FWD = 0, DIR_DGRAD, DIR_WGRAD };

struct ConvLayer {
  int pw;                  // parameter index
  int Co, Ci, Cop, Cip, ksz, stride, T;
  size_t wf_hi, wf_lo;     // packed forward weights   [T][Cop][Cip]
  size_t wd_hi, wd_lo;     // packed data-grad weights [T][Cip][Cop]
  size_t dw;               // fp32 accumulator         [T][Cip][Cop]
  bool need_dgrad;
  LayerKind kind;
  int pb;
  std::string name;        // state-dict key (profiling labels)
};

// How layer c runs in direction dir: everything the ops, the pack jobs and the MAC accounting take from its kind.
struct ConvRole {
  int stride;              // traversal stride on the A operand (the input; dgrad: the output gradient)
  int nopad;               // 1: no padding
  int cls_mode;            // ConvOp::cls_mode
  bool bias;               // + bias parameter pb, the output's high boundary forced to 0 (ConvOp::zero_last)
  int pack;                // PackMode of the weights the op reads; DIR_WGRAD: unpack mode of the accumulator
  bool swap;               // the op sees the layer with Ci and Co exchanged: the data gradient, and the weight gradient of a
                           // kernel = stride layer, which is that of the stride-2 convolution from the fine grid (dU, Co) to the
                           // coarse grid (X, Ci): a = dU, dy = X, accumulator [T][Cop][Cip]
  int macs_div;            // a transposed layer's output grid has 8x the voxels of its input
};

static ConvRole conv_role(const ConvLayer& c, ConvDir dir) {
  const bool up = c.kind != LAYER_CONV, k2 = c.kind == LAYER_CONVT_K2S2;
  ConvRole r = {};
  r.nopad = k2 ? 1 : 0;
  r.bias = dir == DIR_FWD && c.kind == LAYER_CONVT_ZI;
  r.swap = dir == DIR_DGRAD || (dir == DIR_WGRAD && k2);
  r.macs_div = up ? 8 : 1;
  if (dir == DIR_FWD) {
    r.stride = up ? 1 : c.stride;
    r.cls_mode = k2 ? 2 : 0;
    r.pack = k2 ? PACK_T_FWD : up ? PACK_T_FLIPPED : PACK_FWD;
  } else if (dir == DIR_DGRAD) {   // a stride-2 convolution: parity-class mode over the un-inserted output gradient
    r.stride = up ? 2 : 1;
    r.cls_mode = !up && c.stride == 2 ? 1 : 0;
    r.pack = up ? PACK_T_DGRAD : PACK_DGRAD;
  } else {
    r.stride = c.stride;
    r.pack = c.kind == LAYER_CONVT_ZI ? PACK_T_FLIPPED : PACK_FWD;
  }
  return r;
}

struct NormLayer {
  int pg, pb;
  int C, Cld, G;
  long long S;
  size_t coef, coef2, bstats;
  std::string name;
};

struct BlockRec {
  TRef X, a1, y1, a2, out;
  int n1, n2, c1, c2, cs;  // indices into norms / convs (cs = -1 when no sample conv)
  bool first;              // first block of the network: no data gradient in the backward list (input_grad plans: emit_input_grad)
  bool scale_out;          // Dropout3d scale applied to this block's output
  bool scale_in;           // this block's input is the dropout output (its dX must be scaled)
};

struct StageRec {  // decoder up-sampling stage
  TRef Xin;        // raw input of the 1x1x1 pre conv (low res, in_w channels)
  TRef P;          // pre conv output (low res, out_w)
  TRef U;          // up-sampled slice of the concat buffer
  TRef cat;        // full concat view
  int cpre;
  TRef Z;          // transposed-convolution decoder: zero-inserted input (full resolution)
  int cup;         // transposed-convolution layer (-1 in trilinear mode)
};

typedef std::function<int(RunCtx&)> OpFn;

static inline void push_op(std::vector<OpFn>& list, const std::string& label, OpFn fn) {
  list.push_back([label, fn](RunCtx& cx) -> int { cx.label = label.c_str(); return fn(cx); });
}

}  // namespace b200

using namespace b200;

struct b200unet_plan {
  b200unet_net_desc d;
  bool split;
  std::vector<ParamInfo> params;
  std::vector<Buf> bufs;
  std::vector<ConvLayer> convs;
  std::vector<NormLayer> norms;
  std::vector<OpFn> fwd, bwd;
  std::vector<OpFn> igrad;   // input_grad plans: d(loss)/d(x), run by b200unet_plan_input_grad after the backward
  bool input_grad = false;
  size_t cur = 0;
  size_t stats_off = 0, stats_bytes = 0;  // zeroed at the start of every forward
  size_t bz_off = 0, bz_bytes = 0;        // zeroed at the start of every backward (bstats + dw accumulators)
  int last_launches = 0;
  int head_param = -1;
  int head_c = 0;           // channels into the head
  std::vector<PackJob> pack_jobs, unpack_jobs;   // batched weight (un)packing tables (host copies)
  size_t jobs_off = 0;                           // device copy: pack jobs then unpack jobs
  const void* jobs_uploaded_for = nullptr;       // workspace base the table was last uploaded into
  Prof* prof = nullptr;
  double macs[CAT_COUNT] = {0, 0, 0, 0, 0, 0, 0, 0};  // algorithmic MACs per forward+backward pass, by category
  size_t drop_off = 0;      // [N][base_width] floats: copy of the dropout scale of the last forward
  bool have_drop = false;
  bool deterministic = false;   // weight gradients: per-split partial sums + fixed-order reduction instead of fp32 atomics
  size_t head_part_off = 0;   // per-block partial sums of the head weight gradient (fixed-order reduction)
  size_t head_part_bytes = 0;   // at least that, and the transposed-convolution bias gradients' partial sums (run after the head)
  size_t wg_part_off = 0, wg_part_bytes = 0;   // scratch shared by all weight-gradient launches (stream-ordered)
  float slope = 0.f;        // negative slope of the activation (0 = ReLU: UNet3D; 0.01 = LeakyReLU: DynUNet)
  bool infer = false;       // forward-only plan: no backward schedule / buffers, forward temporaries are recycled
  std::vector<std::pair<size_t, std::pair<size_t, size_t>>> free_bufs;   // (bytes, (off_hi, off_lo)) of released buffers

  size_t alloc(size_t bytes) {
    size_t off = (cur + 1023) & ~size_t(1023);
    cur = off + bytes;
    return off;
  }
  int find_param(const std::string& key) const {
    for (size_t i = 0; i < params.size(); ++i)
      if (params[i].key == key) return (int)i;
    return -1;
  }
};

namespace b200 {

typedef b200unet_plan Plan;

static int groups_for(int c, int norm_groups) { return (c < norm_groups || c % norm_groups) ? c : norm_groups; }

static void add_param(Plan& P, const std::string& key, std::initializer_list<int64_t> shp) {
  ParamInfo pi;
  pi.key = key;
  pi.ndim = (int)shp.size();
  int i = 0;
  for (int k = 0; k < 5; ++k) pi.shape[k] = 0;
  for (auto v : shp) pi.shape[i++] = v;
  P.params.push_back(pi);
}

static void add_block_params(Plan& P, const std::string& pre, int cin, int cout) {
  add_param(P, pre + ".conv1.norm1.weight", {cin});
  add_param(P, pre + ".conv1.norm1.bias", {cin});
  add_param(P, pre + ".conv1.conv.weight", {cout, cin, 3, 3, 3});
  add_param(P, pre + ".conv2.norm1.weight", {cout});
  add_param(P, pre + ".conv2.norm1.bias", {cout});
  add_param(P, pre + ".conv2.conv.weight", {cout, cout, 3, 3, 3});
  if (cin != cout) add_param(P, pre + ".sample.weight", {cout, cin, 1, 1, 1});
}

static void dec_widths(const b200unet_net_desc& d, int depth, int* in_w, int* out_w) {
  int L = d.n_levels;
  int o, i;
  if (depth > 0) {
    o = d.base_width;
    for (int k = 0; k < depth - 1; ++k) o *= d.feature_dilation;
    i = o * d.feature_dilation;
  } else {
    o = d.base_width;
    i = d.base_width;
  }
  if (depth != L - 1) i *= 2;
  *in_w = i;
  *out_w = o;
}

static void unet3d_param_spec(Plan& P) {
  const b200unet_net_desc& d = P.d;
  const int L = d.n_levels;
  int cin = d.n_features;
  int w = d.base_width;
  std::vector<int> widths;
  for (int li = 0; li < L; ++li) { widths.push_back(w); w *= d.feature_dilation; }
  for (int li = 0; li < L; ++li) {
    for (int b = 0; b < d.encoder_blocks[li]; ++b)
      add_block_params(P, "encoder.layers." + std::to_string(li) + ".blocks." + std::to_string(b),
                       b == 0 ? cin : widths[li], widths[li]);
    cin = widths[li];
  }
  for (int li = 0; li + 1 < L; ++li)
    add_param(P, "encoder.downsampling_convolutions." + std::to_string(li) + ".weight", {widths[li], widths[li], 3, 3, 3});
  for (int i = 0; i < L; ++i) {
    int depth = L - 1 - i, in_w, out_w;
    dec_widths(d, depth, &in_w, &out_w);
    int planes = depth != 0 ? in_w : out_w;
    for (int b = 0; b < d.decoder_blocks[i]; ++b)
      add_block_params(P, "decoder.layers." + std::to_string(i) + ".blocks." + std::to_string(b), b == 0 ? in_w : planes,
                       planes);
  }
  for (int i = 0; i + 1 < L; ++i) {
    int in_w, out_w;
    dec_widths(d, L - 1 - i, &in_w, &out_w);
    if (d.use_transposed_convolutions) {
      add_param(P, "decoder.upsampling_blocks." + std::to_string(i) + ".weight", {in_w, out_w, 3, 3, 3});
      add_param(P, "decoder.upsampling_blocks." + std::to_string(i) + ".bias", {out_w});
    } else {
      add_param(P, "decoder.pre_upsampling_blocks." + std::to_string(i) + ".weight", {out_w, in_w, 1, 1, 1});
    }
  }
  add_param(P, "final_convolution.weight", {d.n_outputs, d.base_width, 1, 1, 1});
}

// ------------------------------------------------------------------------------------------------ builders
static int new_buf(Plan& P, int N, int D, int H, int W, int C) {
  Buf b;
  size_t bytes = (size_t)N * D * H * W * C * sizeof(bf16);
  bool reused = false;
  for (size_t i = 0; i < P.free_bufs.size(); ++i)
    if (P.free_bufs[i].first == bytes) {   // forward-only plans: take a released buffer of the same size
      b.off_hi = P.free_bufs[i].second.first;
      b.off_lo = P.free_bufs[i].second.second;
      P.free_bufs.erase(P.free_bufs.begin() + i);
      reused = true;
      break;
    }
  if (!reused) {
    b.off_hi = P.alloc(bytes);
    b.off_lo = P.split ? P.alloc(bytes) : 0;
  }
  b.N = N; b.D = D; b.H = H; b.W = W; b.C = C;
  b.stats_off = -1;
  P.bufs.push_back(b);
  return (int)P.bufs.size() - 1;
}

// forward-only plans: the launches are stream-ordered, so a buffer whose last reader has been emitted can back a later
// tensor.  Only whole buffers are released (never a channel slice of a concat buffer while the other half is live).
static void release_buf(Plan& P, int buf) {
  if (!P.infer || buf < 0) return;
  const Buf& b = P.bufs[buf];
  P.free_bufs.push_back({(size_t)b.N * b.D * b.H * b.W * b.C * sizeof(bf16), {b.off_hi, b.off_lo}});
}

static void release_if_whole(Plan& P, TRef t);

static TRef full(const Plan& P, int buf) { TRef t = {buf, 0, P.bufs[buf].C, 0}; return t; }
static TRef slice(TRef t, int c0, int c) { TRef r = {t.buf, t.c0 + c0, c, t.vis_m1}; return r; }
static TRef masked(TRef t) { TRef r = t; r.vis_m1 = 1; return r; }
static void release_if_whole(Plan& P, TRef t) {
  if (t.valid() && t.c0 == 0 && t.c == P.bufs[t.buf].C) release_buf(P, t.buf);
}

static Act act_of(const Plan& P, const RunCtx& cx, TRef t) {
  const Buf& b = P.bufs[t.buf];
  bf16* hi = reinterpret_cast<bf16*>(cx.ws + b.off_hi) + t.c0;
  bf16* lo = P.split ? reinterpret_cast<bf16*>(cx.ws + b.off_lo) + t.c0 : nullptr;
  Act a = make_act(hi, lo, b.N, b.D, b.H, b.W, t.c, b.C);
  if (t.vis_m1) { a.vD = b.D - 1; a.vH = b.H - 1; a.vW = b.W - 1; }
  return a;
}

static void need_stats(Plan& P, int buf) {
  Buf& b = P.bufs[buf];
  if (b.stats_off >= 0) return;
  b.stats_off = (long long)P.stats_bytes;
  P.stats_bytes += ((size_t)b.N * b.C * 2 * sizeof(double) + 255) & ~size_t(255);
}
static double* stats_ptr(const Plan& P, const RunCtx& cx, TRef t) {
  const Buf& b = P.bufs[t.buf];
  return reinterpret_cast<double*>(cx.ws + P.stats_off + b.stats_off) + (size_t)t.c0 * 2;
}

static int new_conv(Plan& P, const std::string& key, int Co, int Ci, int ksz, int stride, bool need_dgrad, LayerKind kind = LAYER_CONV) {
  ConvLayer c;
  c.pw = P.find_param(key);
  c.name = key;
  c.Co = Co; c.Ci = Ci; c.Cop = round_up(Co, 8); c.Cip = round_up(Ci, 8);
  c.ksz = ksz; c.stride = stride; c.T = ksz * ksz * ksz;
  need_dgrad = need_dgrad && !P.infer;
  c.need_dgrad = need_dgrad;
  c.kind = kind;
  c.pb = -1;
  size_t n = (size_t)c.T * c.Cop * c.Cip;
  c.wf_hi = P.alloc(n * 2);
  c.wf_lo = P.split ? P.alloc(n * 2) : 0;
  c.wd_hi = need_dgrad ? P.alloc(n * 2) : 0;
  c.wd_lo = (need_dgrad && P.split) ? P.alloc(n * 2) : 0;
  c.dw = P.bz_bytes;  // relative to bz_off
  if (!P.infer) P.bz_bytes += (n * sizeof(float) + 255) & ~size_t(255);
  P.convs.push_back(c);
  return (int)P.convs.size() - 1;
}

// a norm with G groups over C channels (instance norm: G = C)
static int new_norm(Plan& P, const std::string& prefix, int C, int Cld, long long S, int G) {
  NormLayer n;
  n.name = prefix;
  n.pg = P.find_param(prefix + ".weight");
  n.pb = P.find_param(prefix + ".bias");
  n.C = C; n.Cld = Cld; n.G = G; n.S = S;
  n.coef = P.alloc((size_t)P.d.batch * Cld * 4 * sizeof(float));
  n.coef2 = P.infer ? 0 : P.alloc((size_t)P.d.batch * Cld * 2 * sizeof(float));
  n.bstats = P.bz_bytes;
  if (!P.infer) P.bz_bytes += ((size_t)P.d.batch * Cld * 2 * sizeof(double) + 255) & ~size_t(255);
  P.norms.push_back(n);
  return (int)P.norms.size() - 1;
}

static inline void prof_mark(RunCtx& cx, int cat, bool end) {
  Prof* p = cx.prof;
  if (!p) return;
  if (!end) {
    if ((p->used + 1) * 2 > p->ev.size()) { p->overflow = true; return; }
    p->cat[p->used] = cat;
    p->label[p->used] = cx.label ? cx.label : "";
    cudaEventRecord(p->ev[p->used * 2], cx.st);
  } else {
    if (p->overflow) return;
    cudaEventRecord(p->ev[p->used * 2 + 1], cx.st);
    p->used++;
  }
}
#define LAUNCHED(cx, cat, expr) do { prof_mark(cx, cat, false); B200_TRY(expr); prof_mark(cx, cat, true); (cx).launches++; } while (0)

static std::string shape_of(const Plan& P, TRef t) {
  const Buf& b = P.bufs[t.buf];
  return std::to_string(t.c) + "ch@" + std::to_string(b.D) + "x" + std::to_string(b.H) + "x" + std::to_string(b.W);
}

// ---- forward op emitters (weight packing is batched: see emit_prologue)
static void emit_norm_fwd(Plan& P, int ni, TRef x, TRef y) {
  push_op(P.fwd, "gn_apply " + P.norms[ni].name + " " + shape_of(P, x), [&P, ni, x, y](RunCtx& cx) -> int {
    const NormLayer& n = P.norms[ni];
    // statistics -> coefficients -> normalise + ReLU in one launch (the coefficients are kept for the backward pass)
    LAUNCHED(cx, CAT_NORM, launch_gn_apply(act_of(P, cx, x), act_of(P, cx, y), stats_ptr(P, cx, x), cx.params[n.pg],
                                           cx.params[n.pb], n.C, n.G, n.S, 1e-5f, reinterpret_cast<float*>(cx.ws + n.coef),
                                           P.slope, cx.st));
    return OK;
  });
}

// A operand + packed weights of layer c in direction dir (DIR_FWD or DIR_DGRAD): its forward pack applied to x, or its
// data-gradient pack applied to x = the gradient of its output
static ConvSrc conv_src(const Plan& P, const RunCtx& cx, const ConvLayer& c, TRef x, ConvDir dir) {
  const ConvRole r = conv_role(c, dir);
  const bool dgrad = dir == DIR_DGRAD;
  ConvSrc s;
  memset(&s, 0, sizeof(s));
  s.x = act_of(P, cx, x);
  s.w_hi = reinterpret_cast<bf16*>(cx.ws + (dgrad ? c.wd_hi : c.wf_hi));
  s.w_lo = P.split ? reinterpret_cast<bf16*>(cx.ws + (dgrad ? c.wd_lo : c.wf_lo)) : nullptr;
  s.ksz = c.ksz;
  s.nopad = r.nopad;
  s.stride = r.stride;
  s.Cip = r.swap ? c.Cop : c.Cip;   // K extent: the data-gradient pack [T][Cip][Cop] has Cop
  return s;
}

// the convolution through layer c in direction dir (DIR_FWD or DIR_DGRAD) from x to out, plain epilogue
static ConvOp conv_op(const Plan& P, const RunCtx& cx, const ConvLayer& c, ConvDir dir, TRef x, TRef out) {
  const ConvRole r = conv_role(c, dir);
  ConvOp op;
  memset(&op, 0, sizeof(op));
  op.nsrc = 1;
  op.src[0] = conv_src(P, cx, c, x, dir);
  op.Cop = r.swap ? c.Cip : c.Cop;
  op.out = act_of(P, cx, out);
  op.cls_mode = r.cls_mode;
  if (r.bias) { op.bias = cx.params[c.pb]; op.zero_last = 1; }
  return op;
}

// the weight gradient of layer c from its input a and the gradient dy of its output (Acts of act_of, or of shape_act for sizing)
static WgradOp wgrad_op(const ConvLayer& c, const Act& a, const Act& dy) {
  const ConvRole r = conv_role(c, DIR_WGRAD);
  WgradOp op;
  memset(&op, 0, sizeof(op));
  op.a = r.swap ? dy : a;
  op.dy = r.swap ? a : dy;
  op.ksz = c.ksz; op.stride = r.stride; op.nopad = r.nopad;
  op.Cip = r.swap ? c.Cop : c.Cip;
  op.Cop = r.swap ? c.Cip : c.Cop;
  return op;
}

// algorithmic MACs of layer ci in direction dir; out_like is on the grid of the layer's output
static double conv_macs(const Plan& P, int ci, ConvDir dir, TRef out_like) {
  const ConvLayer& c = P.convs[ci];
  const Buf& b = P.bufs[out_like.buf];
  return (double)b.N * b.D * b.H * b.W * c.Co * c.Ci * c.T / (double)conv_role(c, dir).macs_div;
}

// generic forward-weights conv:  out = (conv(a, W[ci]) [+ conv1x1(a2, W[ci2])] [+ res]) [* dropout]
static void emit_conv_fwd(Plan& P, int ci, TRef a, int ci2, TRef a2, TRef res, TRef out, bool stats, bool scale) {
  if (stats) need_stats(P, out.buf);
  const int cat = CAT_CONV_FWD;
  P.macs[cat] += conv_macs(P, ci, DIR_FWD, out) + (ci2 >= 0 ? conv_macs(P, ci2, DIR_FWD, out) : 0.0);
  push_op(P.fwd, "conv_fwd " + P.convs[ci].name + " " + shape_of(P, a) + "->" + shape_of(P, out) + (ci2 >= 0 ? " +sample" : "") + (res.valid() ? " +res" : ""),
          [&P, ci, a, ci2, a2, res, out, stats, scale, cat](RunCtx& cx) -> int {
    ConvOp op = conv_op(P, cx, P.convs[ci], DIR_FWD, a, out);
    if (ci2 >= 0) {
      op.nsrc = 2;
      op.src[1] = conv_src(P, cx, P.convs[ci2], a2, DIR_FWD);
    }
    Act r;
    if (res.valid()) { r = act_of(P, cx, res); op.res = &r; }
    if (scale && cx.drop) op.scale = cx.drop;
    if (stats) { op.stats = stats_ptr(P, cx, out); op.stats_ld = P.bufs[out.buf].C; }
    LAUNCHED(cx, cat, launch_igemm_conv(op, cx.st));
    return OK;
  });
}

// out = trilinear x2 up-sampling of in [+ skip, in the same pass], and the statistics of out for the norm that reads it
static void emit_upsample2x_fwd(Plan& P, TRef in, TRef out, TRef skip) {
  need_stats(P, out.buf);
  push_op(P.fwd, std::string(skip.valid() ? "upsample2x_fwd+skip " : "upsample2x_fwd ") + shape_of(P, in),
          [&P, in, out, skip](RunCtx& cx) -> int {
    Act sk;
    if (skip.valid()) sk = act_of(P, cx, skip);
    LAUNCHED(cx, CAT_RESAMPLE, launch_upsample2x_fwd(act_of(P, cx, in), act_of(P, cx, out), stats_ptr(P, cx, out), P.bufs[out.buf].C, cx.st,
                                                     skip.valid() ? &sk : nullptr));
    return OK;
  });
}

// ---- backward op emitters
static Act shape_act(const Plan& P, TRef t) {
  const Buf& b = P.bufs[t.buf];
  return make_act(nullptr, nullptr, b.N, b.D, b.H, b.W, t.c, b.C);
}

// runs one weight-gradient op; in deterministic mode through the partial-sum scratch + the fixed-order reduction
static int run_wgrad(Plan& P, RunCtx& cx, WgradOp& op) {
  if (!P.deterministic) {
    LAUNCHED(cx, CAT_CONV_WGRAD, launch_wgrad(op, cx.st));
    return OK;
  }
  int splits = 0;
  op.part = reinterpret_cast<float*>(cx.ws + P.wg_part_off);
  op.part_bytes = P.wg_part_bytes;
  op.part_splits = &splits;
  LAUNCHED(cx, CAT_CONV_WGRAD, launch_wgrad(op, cx.st));
  B200_REQUIRE(splits >= 1, E_INVALID, "plan: internal: deterministic weight gradient wrote no partial slots");
  LAUNCHED(cx, CAT_CONV_WGRAD, launch_wgrad_reduce(op.part, splits, (long long)op.ksz * op.ksz * op.ksz * op.Cip * op.Cop, op.dw, cx.st));
  return OK;
}

// weight gradient of layer ci from its input a and the gradient dy of its output
static void emit_wgrad(Plan& P, int ci, TRef a, TRef dy) {
  P.macs[CAT_CONV_WGRAD] += conv_macs(P, ci, DIR_WGRAD, dy);
  if (P.deterministic)
    P.wg_part_bytes = std::max(P.wg_part_bytes, wgrad_partial_bytes(wgrad_op(P.convs[ci], shape_act(P, a), shape_act(P, dy)), device_sms()));
  push_op(P.bwd, "wgrad " + P.convs[ci].name + " " + shape_of(P, a) + " x " + shape_of(P, dy), [&P, ci, a, dy](RunCtx& cx) -> int {
    const ConvLayer& c = P.convs[ci];
    WgradOp op = wgrad_op(c, act_of(P, cx, a), act_of(P, cx, dy));
    op.dw = reinterpret_cast<float*>(cx.ws + P.bz_off + c.dw);
    return run_wgrad(P, cx, op);
  });
}

// data gradient through layer ci:  out = conv(dy, Wd)  with either the GN/ReLU backward epilogue (ni >= 0, gn_x = raw input of
// the norm) or a plain epilogue (+res, *dropout scale).  reads_input: the layer reads the network input, so its data gradient is
// left out of the algorithmic MACs (b200unet_plan_algorithmic_macs).
static void emit_dgrad(Plan& P, int ci, TRef dy, TRef out, int ni, TRef gn_x, TRef res, bool scale, bool reads_input = false,
                       std::vector<OpFn>* list = nullptr) {
  const int cat = CAT_CONV_DGRAD;
  if (!reads_input) P.macs[cat] += conv_macs(P, ci, DIR_DGRAD, dy);
  push_op(list ? *list : P.bwd, std::string(ni >= 0 ? "dgrad+gnrelu " : "dgrad ") + P.convs[ci].name + " " + shape_of(P, dy) + "->" + shape_of(P, out),
          [&P, ci, dy, out, ni, gn_x, res, scale, cat](RunCtx& cx) -> int {
    ConvOp op = conv_op(P, cx, P.convs[ci], DIR_DGRAD, dy, out);
    Act r, gx;
    if (res.valid()) { r = act_of(P, cx, res); op.res = &r; }
    if (scale && cx.drop) op.scale = cx.drop;
    if (ni >= 0) {
      const NormLayer& n = P.norms[ni];
      op.mode = 1;
      gx = act_of(P, cx, gn_x);
      op.gn_x = &gx;
      op.coef = reinterpret_cast<float*>(cx.ws + n.coef);
      op.coef_ld = n.Cld;
      op.slope = P.slope;
      op.bstats = reinterpret_cast<double*>(cx.ws + P.bz_off + n.bstats);
    }
    LAUNCHED(cx, cat, launch_igemm_conv(op, cx.st));
    return OK;
  });
}

static void emit_gn_bwd_finalize(Plan& P, int ni) {
  push_op(P.bwd, "gn_bwd_finalize " + P.norms[ni].name, [&P, ni](RunCtx& cx) -> int {
    const NormLayer& n = P.norms[ni];
    LAUNCHED(cx, CAT_NORM, launch_gn_bwd_finalize(reinterpret_cast<double*>(cx.ws + P.bz_off + n.bstats),
                                        reinterpret_cast<float*>(cx.ws + n.coef), cx.params[n.pg], P.d.batch, n.C, n.Cld,
                                        n.G, n.S, reinterpret_cast<float*>(cx.ws + n.coef2), cx.grads[n.pg],
                                        cx.grads[n.pb], cx.st));
    return OK;
  });
}

static void emit_gn_bwd(Plan& P, int ni, TRef dz, TRef x, TRef add1, TRef dx, bool scale) {
  push_op(P.bwd, "gn_bwd " + P.norms[ni].name + " " + shape_of(P, x), [&P, ni, dz, x, add1, dx, scale](RunCtx& cx) -> int {
    const NormLayer& n = P.norms[ni];
    Act a1;
    if (add1.valid()) a1 = act_of(P, cx, add1);
    // finalize fused: (E, F), dgamma, dbeta are derived from the backward statistics inside the kernel
    LAUNCHED(cx, CAT_NORM, launch_gn_bwd(act_of(P, cx, dz), act_of(P, cx, x), reinterpret_cast<float*>(cx.ws + n.coef),
                                         reinterpret_cast<double*>(cx.ws + P.bz_off + n.bstats), cx.params[n.pg], n.C, n.G,
                                         n.S, cx.grads[n.pg], cx.grads[n.pb], add1.valid() ? &a1 : nullptr, nullptr,
                                         act_of(P, cx, dx), (scale && cx.drop) ? cx.drop : nullptr, cx.st));
    return OK;
  });
}

// returns the gradient of norm ni's input x from the gradient g1 (+ g2) of its activated output: the activation's backward
// (which also takes the norm's backward statistics), then the norm's
static TRef emit_act_norm_bwd(Plan& P, int ni, TRef x, TRef g1, TRef g2) {
  const Buf xb = P.bufs[x.buf];
  const TRef dz = full(P, new_buf(P, xb.N, xb.D, xb.H, xb.W, x.c));
  push_op(P.bwd, "act_bwd " + P.norms[ni].name + " " + shape_of(P, x), [&P, ni, g1, g2, x, dz](RunCtx& cx) -> int {
    const NormLayer& n = P.norms[ni];
    Act a2;
    if (g2.valid()) a2 = act_of(P, cx, g2);
    LAUNCHED(cx, CAT_NORM, launch_act_bwd(act_of(P, cx, g1), g2.valid() ? &a2 : nullptr, act_of(P, cx, x),
                                          reinterpret_cast<float*>(cx.ws + n.coef), P.slope, act_of(P, cx, dz),
                                          reinterpret_cast<double*>(cx.ws + P.bz_off + n.bstats), n.Cld, cx.st));
    return OK;
  });
  const TRef dx = full(P, new_buf(P, xb.N, xb.D, xb.H, xb.W, x.c));
  emit_gn_bwd(P, ni, dz, x, kNone, dx, false);
  return dx;
}

// dx = the adjoint of the trilinear x2 up-sampling applied to dy
static void emit_upsample2x_bwd(Plan& P, TRef dy, TRef dx) {
  push_op(P.bwd, "upsample2x_bwd " + shape_of(P, dx), [&P, dy, dx](RunCtx& cx) -> int {
    LAUNCHED(cx, CAT_RESAMPLE, launch_upsample2x_bwd(act_of(P, cx, dy), act_of(P, cx, dx), cx.st));
    return OK;
  });
}

// the per-parameter pointers (cx.params or cx.grads) as the batched (un)packing kernels take them
static PtrTable ptr_table(const Plan& P, const float* const* p) {
  PtrTable tbl;
  memset(&tbl, 0, sizeof(tbl));
  for (size_t i = 0; i < P.params.size(); ++i) tbl.p[i] = p[i];
  return tbl;
}

// First op of every forward: zero the statistics arena, upload the job tables into a new workspace, pack all weights (one
// launch) and pack the network input (with_input_stats: and its channel statistics, for a GroupNorm that reads it).  Returns
// the packed input, its channels padded to a multiple of 8.
static TRef emit_prologue(Plan& P, bool with_input_stats) {
  const b200unet_net_desc& d = P.d;
  const int b_in = new_buf(P, d.batch, d.depth, d.height, d.width, round_up(d.n_features, 8));
  if (with_input_stats) need_stats(P, b_in);
  push_op(P.fwd, "pack_weights+input_pack", [&P, b_in, with_input_stats](RunCtx& cx) -> int {
    B200_CHECK_CUDA(cudaMemsetAsync(cx.ws + P.stats_off, 0, P.stats_bytes, cx.st));
    if (P.jobs_uploaded_for != cx.ws) {     // (re)upload the constant job tables into this workspace
      std::vector<PackJob> all(P.pack_jobs);
      all.insert(all.end(), P.unpack_jobs.begin(), P.unpack_jobs.end());
      B200_CHECK_CUDA(cudaMemcpyAsync(cx.ws + P.jobs_off, all.data(), sizeof(PackJob) * all.size(), cudaMemcpyHostToDevice, cx.st));
      B200_CHECK_CUDA(cudaStreamSynchronize(cx.st));   // `all` is a temporary; happens once per workspace
      P.jobs_uploaded_for = cx.ws;
    }
    if (!cx.skip_pack)
      LAUNCHED(cx, CAT_PACK, launch_pack_all(ptr_table(P, cx.params), reinterpret_cast<const PackJob*>(cx.ws + P.jobs_off),
                                             (int)P.pack_jobs.size(), cx.ws, P.split, cx.st));
    TRef t = full(P, b_in);
    LAUNCHED(cx, CAT_RESAMPLE, launch_input_pack(cx.x, P.d.n_features, act_of(P, cx, t), with_input_stats ? stats_ptr(P, cx, t) : nullptr,
                                                 P.bufs[b_in].C, cx.st));
    return OK;
  });
  return full(P, b_in);
}

// The 1x1x1 head (bias_param >= 0: with a bias).  Training plans also get the first op of the backward and the head's backward
// op; *dX = the gradient of Xfinal (kNone in a forward-only plan).  launch_head_fwd / launch_head_bwd pick the kernels from
// n_outputs; above 8 outputs the bias gradient comes out of the same backward pass instead of launch_head_dbias.
static int emit_head(Plan& P, TRef Xfinal, int w_param, int bias_param, TRef* dX) {
  if (!P.infer) {
    // UNet3D's constructor is the one that takes the activation kinds, so its message names them
    B200_REQUIRE(P.d.activation == 0, E_UNSUPPORTED, "plan: activation inside the model%s is inference-only; train on logits",
                 P.d.arch == 0 ? " (sigmoid/softmax)" : "");
    push_op(P.bwd, "memset", [&P](RunCtx& cx) -> int {   // zero the backward statistics and the weight-gradient accumulators
      B200_CHECK_CUDA(cudaMemsetAsync(cx.ws + P.bz_off, 0, P.bz_bytes, cx.st));
      return OK;
    });
  }
  P.head_param = w_param;
  P.head_c = Xfinal.c;
  push_op(P.fwd, "head_fwd", [&P, Xfinal, bias_param](RunCtx& cx) -> int {
    LAUNCHED(cx, CAT_HEAD, launch_head_fwd(act_of(P, cx, Xfinal), cx.params[P.head_param], P.d.n_outputs, P.d.activation, cx.logits, cx.st,
                                           bias_param >= 0 ? cx.params[bias_param] : nullptr));
    return OK;
  });
  *dX = kNone;
  if (P.infer) return OK;
  const Buf xb = P.bufs[Xfinal.buf];
  const TRef g = full(P, new_buf(P, xb.N, xb.D, xb.H, xb.W, Xfinal.c));
  *dX = g;
  push_op(P.bwd, "head_bwd", [&P, Xfinal, g, bias_param](RunCtx& cx) -> int {
    float* scratch = reinterpret_cast<float*>(cx.ws + P.head_part_off);
    const bool fused_dbias = bias_param >= 0 && P.d.n_outputs > 8;
    LAUNCHED(cx, CAT_HEAD, launch_head_bwd(act_of(P, cx, Xfinal), cx.params[P.head_param], P.d.n_outputs, cx.dlogits, act_of(P, cx, g),
                                           cx.grads[P.head_param], cx.st, scratch, fused_dbias ? cx.grads[bias_param] : nullptr));
    if (bias_param >= 0 && !fused_dbias) {
      const Buf& b = P.bufs[Xfinal.buf];
      LAUNCHED(cx, CAT_HEAD, launch_head_dbias(cx.dlogits, b.N, P.d.n_outputs, (long long)b.D * b.H * b.W, cx.grads[bias_param], cx.st,
                                               scratch));
    }
    return OK;
  });
  return OK;
}

// last op of every backward: weight gradients, accumulator -> torch layout (one batched launch)
static void emit_unpack_wgrads(Plan& P) {
  push_op(P.bwd, "unpack_wgrads", [&P](RunCtx& cx) -> int {
    const PackJob* jobs = reinterpret_cast<const PackJob*>(cx.ws + P.jobs_off) + P.pack_jobs.size();
    LAUNCHED(cx, CAT_PACK, launch_unpack_all(ptr_table(P, cx.grads), jobs, (int)P.unpack_jobs.size(), cx.ws, cx.st));
    return OK;
  });
}

// ------------------------------------------------------------------------------------------------ residual block
// state-dict keys of a pre-activation residual block: its two norms (prefixes of .weight / .bias), its two 3x3x3 convolutions
// and the 1x1x1 `sample` convolution it has when it changes the width
struct BlockKeys {
  std::string n1, c1, n2, c2, sample;
};
static BlockKeys unet3d_block_keys(const std::string& pre) {   // classification/myronenko.py:34-58
  return {pre + ".conv1.norm1", pre + ".conv1.conv.weight", pre + ".conv2.norm1", pre + ".conv2.conv.weight", pre + ".sample.weight"};
}

static BlockRec build_block_fwd(Plan& P, const BlockKeys& k, TRef X, int cin_real, int C, TRef dest, bool want_stats,
                                bool first, bool scale_out, bool scale_in, bool x_dead) {
  const Buf& xb = P.bufs[X.buf];
  const int N = xb.N, D = xb.D, H = xb.H, W = xb.W;
  const long long S = (long long)D * H * W;
  BlockRec r;
  r.X = X; r.first = first; r.scale_out = scale_out; r.scale_in = scale_in;
  r.n1 = new_norm(P, k.n1, cin_real, X.c, S, groups_for(cin_real, P.d.norm_groups));
  r.c1 = new_conv(P, k.c1, C, cin_real, 3, 1, true);
  r.n2 = new_norm(P, k.n2, C, C, S, groups_for(C, P.d.norm_groups));
  r.c2 = new_conv(P, k.c2, C, C, 3, 1, true);
  r.cs = (cin_real != C) ? new_conv(P, k.sample, C, cin_real, 1, 1, !first || P.input_grad) : -1;
  r.a1 = full(P, new_buf(P, N, D, H, W, X.c));
  r.y1 = full(P, new_buf(P, N, D, H, W, C));
  r.a2 = full(P, new_buf(P, N, D, H, W, C));
  r.out = dest;
  emit_norm_fwd(P, r.n1, X, r.a1);
  emit_conv_fwd(P, r.c1, r.a1, -1, kNone, kNone, r.y1, true, false);
  emit_norm_fwd(P, r.n2, r.y1, r.a2);
  if (r.cs >= 0) emit_conv_fwd(P, r.c2, r.a2, r.cs, X, kNone, dest, want_stats, scale_out);
  else emit_conv_fwd(P, r.c2, r.a2, -1, kNone, X, dest, want_stats, scale_out);
  release_buf(P, r.a1.buf);
  release_buf(P, r.y1.buf);
  release_buf(P, r.a2.buf);
  if (x_dead) release_if_whole(P, X);
  return r;
}

// input_grad plans: d(loss)/d(x) -> NCDHW fp32 from the first block's gradients (UNet3D: dz = the data gradient of its conv1
// through the GroupNorm/ReLU epilogue, x = the packed network input, norm ni; r = the residual branch's gradient.  DynUNet: ni < 0,
// r = the data gradient of input_block.conv1).  Backward buffers are never recycled in a training plan, so dz, x and r still hold
// what the backward left in them.
static void emit_input_grad(Plan& P, int ni, TRef dz, TRef x, TRef r) {
  push_op(P.igrad, "input_grad " + shape_of(P, r), [&P, ni, dz, x, r](RunCtx& cx) -> int {
    if (ni < 0) {
      LAUNCHED(cx, CAT_RESAMPLE, launch_input_grad(nullptr, nullptr, nullptr, nullptr, 0, act_of(P, cx, r), P.d.n_features, cx.dx, cx.st));
      return OK;
    }
    const NormLayer& n = P.norms[ni];
    const Act a = act_of(P, cx, dz), b = act_of(P, cx, x);
    LAUNCHED(cx, CAT_NORM, launch_input_grad(&a, &b, reinterpret_cast<const float*>(cx.ws + n.coef), reinterpret_cast<const float*>(cx.ws + n.coef2),
                                             n.Cld, act_of(P, cx, r), P.d.n_features, cx.dx, cx.st));
    return OK;
  });
}

// input_grad plans: the data gradient of layer ci, which reads the packed network input x, from the gradient dy of its output,
// then d(loss)/d(x) from it (ni, dz: see emit_input_grad)
static void emit_input_dgrad(Plan& P, int ci, TRef dy, TRef x, int ni, TRef dz) {
  const Buf xb = P.bufs[x.buf];
  const TRef r = full(P, new_buf(P, xb.N, xb.D, xb.H, xb.W, x.c));
  emit_dgrad(P, ci, dy, r, -1, kNone, kNone, false, /*reads_input=*/true, &P.igrad);
  emit_input_grad(P, ni, dz, x, r);
}

// backward through an encoder's stride-2 convolution ci from the gradient dy of its output: its weight gradient; returns the
// gradient of its input x (also a skip) = the parity-class data gradient + dskip [* the Dropout3d scale].  Parity-class mode:
// eight implicit GEMMs over the un-inserted gradient (27 tap products instead of 8 x 27), TMA-stored into their interleaved positions.
static TRef emit_down_bwd(Plan& P, int ci, TRef x, TRef dy, TRef dskip, bool scale) {
  emit_wgrad(P, ci, x, dy);
  const Buf xb = P.bufs[x.buf];
  const TRef dx = full(P, new_buf(P, xb.N, xb.D, xb.H, xb.W, x.c));
  emit_dgrad(P, ci, dy, dx, -1, kNone, dskip, scale);
  return dx;
}

// returns the TRef of dX (kNone for the first block of the network)
static TRef build_block_bwd(Plan& P, const BlockRec& r, TRef dOut) {
  const Buf& xb = P.bufs[r.X.buf];
  const int N = xb.N, D = xb.D, H = xb.H, W = xb.W;
  const int C = r.y1.c;
  emit_wgrad(P, r.c2, r.a2, dOut);
  if (r.cs >= 0) emit_wgrad(P, r.cs, r.X, dOut);
  TRef dz2 = full(P, new_buf(P, N, D, H, W, C));
  emit_dgrad(P, r.c2, dOut, dz2, r.n2, r.y1, kNone, false);
  TRef dy1 = full(P, new_buf(P, N, D, H, W, C));
  emit_gn_bwd(P, r.n2, dz2, r.y1, kNone, dy1, false);
  emit_wgrad(P, r.c1, r.a1, dy1);
  TRef dz1 = full(P, new_buf(P, N, D, H, W, r.X.c));
  emit_dgrad(P, r.c1, dy1, dz1, r.n1, r.X, kNone, false, /*reads_input=*/r.first);
  if (r.first) {   // no data gradient below the first block: only dgamma / dbeta of its first norm are needed
    emit_gn_bwd_finalize(P, r.n1);
    if (P.input_grad) {
      // dOut already carries the Dropout3d scale of this block's output (applied by whoever produced it): not applied again
      if (r.cs >= 0) emit_input_dgrad(P, r.cs, dOut, r.X, r.n1, dz1);
      else emit_input_grad(P, r.n1, dz1, r.X, dOut);
    }
    return kNone;
  }
  TRef dX = full(P, new_buf(P, N, D, H, W, r.X.c));
  if (r.cs >= 0) {
    emit_gn_bwd(P, r.n1, dz1, r.X, kNone, dX, false);
    emit_dgrad(P, r.cs, dOut, dX, -1, kNone, dX, r.scale_in);  // dX = (conv1x1(dOut, Ws^T) + dX) [* scale]
  } else {
    emit_gn_bwd(P, r.n1, dz1, r.X, dOut, dX, r.scale_in);
  }
  return dX;
}

static int finish_build(Plan& P);

// spatial extents of each level (level 0: the input's), halved from one level to the next
static int level_extents(const b200unet_net_desc& d, std::vector<int>& Ds, std::vector<int>& Hs, std::vector<int>& Ws) {
  const int L = d.n_levels;
  int D = d.depth, H = d.height, W = d.width;
  for (int li = 0; li < L; ++li) {
    Ds.push_back(D); Hs.push_back(H); Ws.push_back(W);
    if (li + 1 < L)
      B200_REQUIRE(D % 2 == 0 && H % 2 == 0 && W % 2 == 0 && D >= 2 && H >= 2 && W >= 2, E_UNSUPPORTED,
                   "plan: level %d extent %dx%dx%d must be even (input %dx%dx%d not divisible by 2^%d)", li, D, H, W,
                   d.depth, d.height, d.width, L - 1);
    D /= 2; H /= 2; W /= 2;
  }
  return OK;
}

static int build_unet3d(Plan& P) {
  const b200unet_net_desc& d = P.d;
  const int L = d.n_levels, N = d.batch;
  B200_REQUIRE(L >= 2 && L <= 8, E_UNSUPPORTED, "plan: n_levels=%d unsupported (2..8)", L);
  B200_REQUIRE(d.base_width % 8 == 0, E_UNSUPPORTED, "plan: base_width=%d must be a multiple of 8", d.base_width);
  B200_REQUIRE(d.n_features >= 1 && d.n_features <= 16, E_UNSUPPORTED, "plan: n_features=%d unsupported", d.n_features);
  B200_REQUIRE(d.n_outputs >= 1 && d.n_outputs <= B200_HEAD_MAX_OUTPUTS, E_UNSUPPORTED, "plan: n_outputs=%d unsupported (1..%d)",
               d.n_outputs, B200_HEAD_MAX_OUTPUTS);
  std::vector<int> widths, Ds, Hs, Ws;
  B200_TRY(level_extents(d, Ds, Hs, Ws));
  for (int li = 0, w = d.base_width; li < L; ++li, w *= d.feature_dilation) widths.push_back(w);
  unet3d_param_spec(P);

  // ---------------- forward
  TRef X = emit_prologue(P, /*with_input_stats=*/true);
  std::vector<std::vector<BlockRec>> enc(L), dec(L);
  std::vector<int> cat(L, -1), down(L, -1);
  std::vector<TRef> skip(L), down_out(L);
  std::vector<StageRec> stages;
  for (int li = 0; li + 1 < L; ++li) {
    cat[li] = new_buf(P, N, Ds[li], Hs[li], Ws[li], 2 * widths[li]);
    need_stats(P, cat[li]);
  }
  int cin_real = d.n_features;
  for (int li = 0; li < L; ++li) {
    const int C = widths[li];
    const int nb = d.encoder_blocks[li];
    B200_REQUIRE(nb >= 1, E_INVALID, "plan: encoder_blocks[%d]=%d", li, nb);
    for (int b = 0; b < nb; ++b) {
      const bool last = (b == nb - 1);
      TRef dest;
      bool want_stats;
      if (last && li + 1 < L) { dest = slice(full(P, cat[li]), C, C); want_stats = true; }
      else { dest = full(P, new_buf(P, N, Ds[li], Hs[li], Ws[li], C)); want_stats = true; }
      const bool first = (li == 0 && b == 0);
      enc[li].push_back(build_block_fwd(P, unet3d_block_keys("encoder.layers." + std::to_string(li) + ".blocks." + std::to_string(b)), X,
                                        cin_real, C, dest, want_stats, first, /*scale_out=*/first,
                                        /*scale_in=*/(li == 0 && b == 1), /*x_dead=*/true));
      X = dest;
      cin_real = C;
    }
    skip[li] = X;
    if (li + 1 < L) {
      down[li] = new_conv(P, "encoder.downsampling_convolutions." + std::to_string(li) + ".weight", C, C, 3, 2, true);
      down_out[li] = full(P, new_buf(P, N, Ds[li + 1], Hs[li + 1], Ws[li + 1], C));
      emit_conv_fwd(P, down[li], X, -1, kNone, kNone, down_out[li], true, false);
      X = down_out[li];
    }
  }
  // decoder
  for (int i = 0; i + 1 < L; ++i) {
    const int depth = L - 1 - i;
    int in_w, out_w;
    dec_widths(d, depth, &in_w, &out_w);
    B200_REQUIRE(in_w == X.c, E_INVALID, "plan: decoder stage %d expects %d channels, has %d", i, in_w, X.c);
    const Buf xb = P.bufs[X.buf];
    for (int b = 0; b < d.decoder_blocks[i]; ++b) {
      TRef dest = full(P, new_buf(P, N, xb.D, xb.H, xb.W, in_w));
      dec[i].push_back(build_block_fwd(P, unet3d_block_keys("decoder.layers." + std::to_string(i) + ".blocks." + std::to_string(b)), X, in_w,
                                       in_w, dest, /*want_stats=*/b + 1 < d.decoder_blocks[i], false, false, false, true));
      X = dest;
    }
    const int j = L - 2 - i;
    B200_REQUIRE(out_w == widths[j], E_INVALID, "plan: decoder stage %d width mismatch", i);
    StageRec s;
    s.Xin = X;
    s.cat = full(P, cat[j]);
    s.U = slice(s.cat, 0, out_w);
    s.cpre = -1; s.cup = -1; s.P = kNone; s.Z = kNone;
    if (!d.use_transposed_convolutions) {
      s.cpre = new_conv(P, "decoder.pre_upsampling_blocks." + std::to_string(i) + ".weight", out_w, in_w, 1, 1, true);
      s.P = full(P, new_buf(P, N, xb.D, xb.H, xb.W, out_w));
      emit_conv_fwd(P, s.cpre, X, -1, kNone, kNone, s.P, false, false);
      release_if_whole(P, X);
      emit_upsample2x_fwd(P, s.P, s.U, kNone);
      release_buf(P, s.P.buf);
    } else {
      // ConvTranspose3d(k3, s2, p1) + bias, then F.pad(+1 high side) = zero-insert + 3x3x3 conv with the flipped
      // kernel over a 2n grid whose last plane/row/column is forced to 0 (decoder.py:101-102, unet.py:34-40)
      const std::string key = "decoder.upsampling_blocks." + std::to_string(i);
      s.cup = new_conv(P, key + ".weight", out_w, in_w, 3, 1, true, LAYER_CONVT_ZI);
      P.convs[s.cup].pb = P.find_param(key + ".bias");
      B200_REQUIRE(P.convs[s.cup].pb >= 0, E_INVALID, "plan: internal: missing bias for %s", key.c_str());
      s.Z = full(P, new_buf(P, N, 2 * xb.D, 2 * xb.H, 2 * xb.W, in_w));
      TRef Xi = X, Z = s.Z;
      push_op(P.fwd, "zero_insert " + shape_of(P, Z), [&P, Xi, Z](RunCtx& cx) -> int {
        LAUNCHED(cx, CAT_RESAMPLE, launch_zero_insert(act_of(P, cx, Xi), act_of(P, cx, Z), 0, 0, 0, cx.st));
        return OK;
      });
      release_if_whole(P, X);
      emit_conv_fwd(P, s.cup, s.Z, -1, kNone, kNone, s.U, true, false);
      release_buf(P, s.Z.buf);
    }
    stages.push_back(s);
    X = s.cat;
  }
  // final stage (depth 0)
  {
    const Buf xb = P.bufs[X.buf];
    int cin = X.c;
    for (int b = 0; b < d.decoder_blocks[L - 1]; ++b) {
      TRef dest = full(P, new_buf(P, N, xb.D, xb.H, xb.W, d.base_width));
      dec[L - 1].push_back(build_block_fwd(P, unet3d_block_keys("decoder.layers." + std::to_string(L - 1) + ".blocks." + std::to_string(b)), X,
                                           cin, d.base_width, dest, b + 1 < d.decoder_blocks[L - 1], false, false, false, true));
      X = dest;
      cin = d.base_width;
    }
  }
  TRef g;
  B200_TRY(emit_head(P, X, P.find_param("final_convolution.weight"), -1, &g));
  if (P.infer) return finish_build(P);

  // ---------------- backward
  for (int b = d.decoder_blocks[L - 1] - 1; b >= 0; --b) g = build_block_bwd(P, dec[L - 1][b], g);
  std::vector<TRef> dskip_dec(L, kNone);
  for (int i = L - 2; i >= 0; --i) {
    const StageRec& s = stages[i];
    const int j = L - 2 - i;
    const int out_w = s.U.c;
    dskip_dec[j] = slice(g, out_w, out_w);
    TRef dU = slice(g, 0, out_w);
    const Buf xb = P.bufs[s.Xin.buf];
    TRef gX = full(P, new_buf(P, N, xb.D, xb.H, xb.W, s.Xin.c));
    if (s.cup < 0) {
      TRef dP = full(P, new_buf(P, N, xb.D, xb.H, xb.W, out_w));
      emit_upsample2x_bwd(P, dU, dP);
      emit_wgrad(P, s.cpre, s.Xin, dP);
      emit_dgrad(P, s.cpre, dP, gX, -1, kNone, kNone, false);
    } else {
      // the padded boundary of the ConvT output is a constant: mask it out of dU (visible extent 2n-1 through TMA)
      TRef dUm = masked(dU);
      const int cup = s.cup;
      P.head_part_bytes = std::max(P.head_part_bytes, bias_grad_scratch_bytes(out_w));
      push_op(P.bwd, "bias_grad " + P.convs[cup].name, [&P, dUm, cup](RunCtx& cx) -> int {
        LAUNCHED(cx, CAT_OTHER, launch_bias_grad(act_of(P, cx, dUm), cx.grads[P.convs[cup].pb],
                                                 reinterpret_cast<float*>(cx.ws + P.head_part_off), cx.st));
        return OK;
      });
      emit_wgrad(P, cup, s.Z, dUm);                                   // dW[tap][ci][co] from the zero-inserted input
      emit_dgrad(P, cup, dUm, gX, -1, kNone, kNone, false);   // stride-2 conv of dU: dX[i] = sum_k dU[2i+k-1] W[ci][co][k]
    }
    for (int b = d.decoder_blocks[i] - 1; b >= 0; --b) gX = build_block_bwd(P, dec[i][b], gX);
    g = gX;
  }
  // g = gradient w.r.t. the bottleneck output (skip[L-1])
  for (int li = L - 1; li >= 0; --li) {
    for (int b = d.encoder_blocks[li] - 1; b >= 0; --b) g = build_block_bwd(P, enc[li][b], g);
    if (li > 0) {
      const int lj = li - 1;
      // dropout scale belongs to the output of encoder block (0,0): that is this tensor iff level 0 has one block
      g = emit_down_bwd(P, down[lj], skip[lj], g, dskip_dec[lj], /*scale=*/lj == 0 && d.encoder_blocks[0] == 1);
    }
  }
  emit_unpack_wgrads(P);
  return finish_build(P);
}

// arenas that are bulk-zeroed + the weight (un)packing job tables
static int finish_build(Plan& P) {
  const b200unet_net_desc& d = P.d;
  const int N = d.batch;
  B200_REQUIRE(P.params.size() <= 256, E_UNSUPPORTED, "plan: more than 256 parameter tensors");
  P.drop_off = P.alloc(sizeof(float) * N * (d.base_width > 0 ? d.base_width : 8));
  P.stats_off = P.alloc(P.stats_bytes);
  P.bz_off = P.alloc(P.bz_bytes);
  if (P.wg_part_bytes) P.wg_part_off = P.alloc(P.wg_part_bytes);
  B200_REQUIRE(d.n_outputs <= 8 || P.head_c <= 64, E_UNSUPPORTED,
               "plan: more than 8 outputs need at most 64 channels into the head, got %d", P.head_c);
  if (!P.infer) P.head_part_off = P.alloc(std::max(P.head_part_bytes, head_bwd_scratch_bytes(d.n_outputs, P.head_c)));
  for (size_t i = 0; i < P.convs.size(); ++i)
    B200_REQUIRE(P.convs[i].pw >= 0, E_INVALID, "plan: internal: conv %d has no parameter", (int)i);
  for (const ConvLayer& c : P.convs) {
    PackJob j;
    j.pidx = c.pw; j.Co = c.Co; j.Ci = c.Ci; j.Cop = c.Cop; j.Cip = c.Cip; j.T = c.T;
    j.mode = conv_role(c, DIR_FWD).pack; j.off_hi = (long long)c.wf_hi; j.off_lo = (long long)c.wf_lo;
    P.pack_jobs.push_back(j);
    if (c.need_dgrad) {
      j.mode = conv_role(c, DIR_DGRAD).pack; j.off_hi = (long long)c.wd_hi; j.off_lo = (long long)c.wd_lo;
      P.pack_jobs.push_back(j);
    }
    if (P.infer) continue;
    const ConvRole r = conv_role(c, DIR_WGRAD);
    PackJob u = j;
    u.mode = r.pack; u.off_hi = (long long)(P.bz_off + c.dw); u.off_lo = 0;
    if (r.swap) { std::swap(u.Co, u.Ci); std::swap(u.Cop, u.Cip); }   // accumulated as [T][Cop][Cip]: reads back as [Ci][Co][T]
    P.unpack_jobs.push_back(u);
  }
  P.jobs_off = P.alloc(sizeof(PackJob) * (P.pack_jobs.size() + P.unpack_jobs.size()));
  return OK;
}


// ================================================================================================ DynUNet (MONAI) blocks
// What examples/brats2020/brats2020_config.json:2-107 and examples/sppin/sppin_config.json train.  MONAI's source is not
// under /root/reference (third-party, absent from this image): the block semantics below restate its public definition
// (monai/networks/nets/dynunet.py, monai/networks/blocks/dynunet_block.py) -- parity unpinned, see oracle/dynunet_oracle.py.
//   UnetBasicBlock(in, out, k3, stride):  conv(bias-free, stride) -> InstanceNorm(affine) -> LeakyReLU(0.01)
//                                         -> conv(s1) -> InstanceNorm -> LeakyReLU                  (post-activation order)
//   UnetUpBlock(in, out):                 ConvTranspose3d(in -> out, kernel = stride = 2, bias-free) -> cat(up, skip) -> UnetBasicBlock(2 out -> out)
//   UnetOutBlock:                         1x1x1 conv with bias
//   DynUNet.forward: input_block, downsamples[...], bottleneck (strides 1, 2, 2, ...), upsamples mirrored, output_block.
struct DynBlock {
  TRef X;            // block input (activated output of the producer, or the concat buffer / packed network input)
  TRef c1, a1, c2;   // conv1 output, its activated norm, conv2 output
  TRef out;          // activated norm of c2 (may be the skip half of a concat buffer)
  int n1, n2, k1, k2;
  int stride;
  bool first;
};

static void add_dyn_block_params(Plan& P, const std::string& pre, int cin, int cout) {
  add_param(P, pre + ".conv1.conv.weight", {cout, cin, 3, 3, 3});
  add_param(P, pre + ".conv2.conv.weight", {cout, cout, 3, 3, 3});
  add_param(P, pre + ".norm1.weight", {cout});
  add_param(P, pre + ".norm1.bias", {cout});
  add_param(P, pre + ".norm2.weight", {cout});
  add_param(P, pre + ".norm2.bias", {cout});
}

// module name of encoder level i of an L-level DynUNet
static std::string dyn_enc_name(int L, int i) {
  return i == 0 ? "input_block" : i == L - 1 ? "bottleneck" : "downsamples." + std::to_string(i - 1);
}

// in MONAI's registration order: input_block, downsamples, bottleneck, upsamples, output_block
static void dynunet_param_spec(Plan& P) {
  const b200unet_net_desc& d = P.d;
  const int L = d.n_levels;
  const int* F = d.filters;
  for (int i = 0; i < L; ++i) add_dyn_block_params(P, dyn_enc_name(L, i), i == 0 ? d.n_features : F[i - 1], F[i]);
  for (int u = 0; u + 1 < L; ++u) {      // upsamples[u] maps level L-1-u -> L-2-u
    const int lo = L - 1 - u, hi = L - 2 - u;
    const std::string pre = "upsamples." + std::to_string(u);
    add_param(P, pre + ".transp_conv.conv.weight", {F[lo], F[hi], 2, 2, 2});
    add_dyn_block_params(P, pre + ".conv_block", 2 * F[hi], F[hi]);
  }
  add_param(P, "output_block.conv.conv.weight", {d.n_outputs, F[0], 1, 1, 1});
  add_param(P, "output_block.conv.conv.bias", {d.n_outputs});
}

static DynBlock build_dyn_block_fwd(Plan& P, const std::string& pre, TRef X, int cin_real, int C, int stride, TRef dest, bool first,
                                    bool x_dead) {
  const Buf& xb = P.bufs[X.buf];
  const int N = xb.N, D = xb.D / stride, H = xb.H / stride, W = xb.W / stride;
  const long long S = (long long)D * H * W;
  DynBlock r;
  r.X = X; r.stride = stride; r.first = first;
  r.k1 = new_conv(P, pre + ".conv1.conv.weight", C, cin_real, 3, stride, !first || P.input_grad);
  r.k2 = new_conv(P, pre + ".conv2.conv.weight", C, C, 3, 1, true);
  r.n1 = new_norm(P, pre + ".norm1", C, C, S, C);
  r.n2 = new_norm(P, pre + ".norm2", C, C, S, C);
  r.c1 = full(P, new_buf(P, N, D, H, W, C));
  emit_conv_fwd(P, r.k1, X, -1, kNone, kNone, r.c1, true, false);
  if (x_dead) release_if_whole(P, X);
  r.a1 = full(P, new_buf(P, N, D, H, W, C));
  emit_norm_fwd(P, r.n1, r.c1, r.a1);
  r.c2 = full(P, new_buf(P, N, D, H, W, C));
  emit_conv_fwd(P, r.k2, r.a1, -1, kNone, kNone, r.c2, true, false);
  r.out = dest;
  emit_norm_fwd(P, r.n2, r.c2, dest);
  release_buf(P, r.c1.buf);
  release_buf(P, r.a1.buf);
  release_buf(P, r.c2.buf);
  return r;
}

// gradient of the block output arrives as g1 (+ g2); returns dX (kNone for the first block)
static TRef build_dyn_block_bwd(Plan& P, const DynBlock& r, TRef g1, TRef g2) {
  const Buf& cb = P.bufs[r.c1.buf];
  const int N = cb.N, D = cb.D, H = cb.H, W = cb.W, C = r.c1.c;
  TRef dc2 = emit_act_norm_bwd(P, r.n2, r.c2, g1, g2);
  emit_wgrad(P, r.k2, r.a1, dc2);
  TRef dz1 = full(P, new_buf(P, N, D, H, W, C));
  emit_dgrad(P, r.k2, dc2, dz1, r.n1, r.c1, kNone, false);   // mode 1: masked by act'(norm1(c1)) + statistics
  TRef dc1 = full(P, new_buf(P, N, D, H, W, C));
  emit_gn_bwd(P, r.n1, dz1, r.c1, kNone, dc1, false);
  emit_wgrad(P, r.k1, r.X, dc1);
  if (r.first) {
    if (P.input_grad) emit_input_dgrad(P, r.k1, dc1, r.X, -1, kNone);
    return kNone;
  }
  const Buf& xb = P.bufs[r.X.buf];
  TRef dX = full(P, new_buf(P, N, xb.D, xb.H, xb.W, r.X.c));
  emit_dgrad(P, r.k1, dc1, dX, -1, kNone, kNone, false);
  return dX;
}

static int build_dynunet(Plan& P) {
  const b200unet_net_desc& d = P.d;
  const int L = d.n_levels, N = d.batch;
  B200_REQUIRE(L >= 2 && L <= 8, E_UNSUPPORTED, "plan: DynUNet with %d levels unsupported (2..8)", L);
  B200_REQUIRE(d.n_features >= 1 && d.n_features <= 16, E_UNSUPPORTED, "plan: in_channels=%d unsupported", d.n_features);
  B200_REQUIRE(d.n_outputs >= 1 && d.n_outputs <= B200_HEAD_MAX_OUTPUTS, E_UNSUPPORTED, "plan: out_channels=%d unsupported (1..%d)",
               d.n_outputs, B200_HEAD_MAX_OUTPUTS);
  std::vector<int> F, Ds, Hs, Ws;
  for (int i = 0; i < L; ++i) {
    B200_REQUIRE(d.filters[i] >= 8 && d.filters[i] % 8 == 0, E_UNSUPPORTED, "plan: filters[%d]=%d must be a positive multiple of 8", i,
                 d.filters[i]);
    F.push_back(d.filters[i]);
  }
  B200_TRY(level_extents(d, Ds, Hs, Ws));
  dynunet_param_spec(P);

  // ---- forward
  TRef X = emit_prologue(P, /*with_input_stats=*/false);
  std::vector<int> cat(L, -1);
  for (int i = 0; i + 1 < L; ++i) cat[i] = new_buf(P, N, Ds[i], Hs[i], Ws[i], 2 * F[i]);
  std::vector<DynBlock> enc(L), dec(L);
  std::vector<int> up(L, -1);
  int cin_real = d.n_features;
  for (int i = 0; i < L; ++i) {
    TRef dest = (i + 1 < L) ? slice(full(P, cat[i]), F[i], F[i]) : full(P, new_buf(P, N, Ds[i], Hs[i], Ws[i], F[i]));
    enc[i] = build_dyn_block_fwd(P, dyn_enc_name(L, i), X, cin_real, F[i], i == 0 ? 1 : 2, dest, i == 0, /*x_dead=*/i == 0);
    X = dest;
    cin_real = F[i];
  }
  for (int u = 0; u + 1 < L; ++u) {
    const int lo = L - 1 - u, hi = L - 2 - u;
    const std::string pre = "upsamples." + std::to_string(u);
    up[hi] = new_conv(P, pre + ".transp_conv.conv.weight", F[hi], F[lo], 2, 2, true, LAYER_CONVT_K2S2);
    emit_conv_fwd(P, up[hi], X, -1, kNone, kNone, slice(full(P, cat[hi]), 0, F[hi]), false, false);
    release_if_whole(P, X);
    TRef dest = full(P, new_buf(P, N, Ds[hi], Hs[hi], Ws[hi], F[hi]));
    dec[hi] = build_dyn_block_fwd(P, pre + ".conv_block", full(P, cat[hi]), 2 * F[hi], F[hi], 1, dest, false, /*x_dead=*/true);
    X = dest;
  }
  TRef g;
  B200_TRY(emit_head(P, X, P.find_param("output_block.conv.conv.weight"), P.find_param("output_block.conv.conv.bias"), &g));
  if (P.infer) return finish_build(P);

  // ---- backward
  std::vector<TRef> dskip(L, kNone);
  for (int hi = 0; hi + 1 < L; ++hi) {     // decoder, top (level 0) to bottom
    const int lo = hi + 1;
    TRef dCat = build_dyn_block_bwd(P, dec[hi], g, kNone);
    dskip[hi] = slice(dCat, F[hi], F[hi]);
    TRef dU = slice(dCat, 0, F[hi]);
    // input of the transposed convolution: the activated output of the stage below (or of the bottleneck)
    const TRef Xlow = (lo == L - 1) ? enc[lo].out : dec[lo].out;
    // dW[ci][co][t] = sum_j X[j][ci] dU[2j + t][co]
    emit_wgrad(P, up[hi], Xlow, dU);
    const Buf lb = P.bufs[Xlow.buf];
    TRef gX = full(P, new_buf(P, N, lb.D, lb.H, lb.W, F[lo]));
    // dX[j][ci] = sum_t sum_co dU[2j + t][co] W[ci][co][t]: a kernel-2 stride-2 unpadded convolution of dU
    emit_dgrad(P, up[hi], dU, gX, -1, kNone, kNone, false);
    g = gX;
  }
  // g = gradient of the bottleneck output; encoder, bottom to top: skip gradient + gradient through the stride-2 conv below
  TRef gdown = kNone;
  for (int i = L - 1; i >= 0; --i) {
    TRef g1 = (i == L - 1) ? g : dskip[i];
    TRef g2 = (i == L - 1) ? kNone : gdown;
    gdown = build_dyn_block_bwd(P, enc[i], g1, g2);
  }
  emit_unpack_wgrads(P);
  return finish_build(P);
}

// ================================================================================================ SegResNet (MONAI)
// MONAI's SegResNet (Myronenko's BraTS 2018 network), absent from this image like DynUNet: restated from its public definition
// (monai/networks/nets/segresnet.py, monai/networks/blocks/segresnet_block.py) -- parity unpinned, see oracle/segresnet_oracle.py.
//   conv(ci, co, k = 3, s = 1, bias = False):  Conv3d, padding k // 2;  F = init_filters, L = len(blocks_down)
//   ResBlock(C):   y = conv2(act(norm2(conv1(act(norm1(x)))))) + x,  GroupNorm(num_groups, C) affine eps 1e-5, C -> C 3x3x3 convs
//   forward:       x = convInit(x) [-> Dropout3d(dropout_prob)];  level i: x = pre_conv_i(x) (Identity at i = 0, else conv(F 2^(i-1),
//                  F 2^i, 3, stride 2)), then blocks_down[i] x ResBlock(F 2^i); down_x[i] = x.  Up stage i = 0..L-2, C = F 2^(L-2-i):
//                  x = upsample2x(conv1x1(2C -> C)(x)) + down_x[L-2-i], then blocks_up[i] x ResBlock(C).
//                  Head: conv_final = GroupNorm(F) -> act -> conv(F, out_channels, 1, bias = True).
//   state dict (registration order): convInit.conv.weight; down_layers.{i}.0.conv.weight (i > 0), down_layers.{i}.{1..}.<ResBlock>;
//                  up_layers.{i}.{0..}.<ResBlock>; up_samples.{i}.0.conv.weight [C, 2C, 1, 1, 1]; conv_final.0.weight / .bias,
//                  conv_final.2.conv.weight / .bias.  <ResBlock> = norm1.weight, norm1.bias, norm2.weight, norm2.bias,
//                  conv1.conv.weight, conv2.conv.weight.
// Schedule: every op is one the UNet3D / DynUNet plans already run, except the up-sampling, which adds the skip in the same pass
// (launch_upsample2x_fwd with an addend) and takes the statistics of the sum for the next ResBlock's norm1.
static BlockKeys segres_block_keys(const std::string& pre) {
  return {pre + ".norm1", pre + ".conv1.conv.weight", pre + ".norm2", pre + ".conv2.conv.weight", pre + ".sample"};
}

static void add_segres_block_params(Plan& P, const std::string& pre, int C) {
  add_param(P, pre + ".norm1.weight", {C});
  add_param(P, pre + ".norm1.bias", {C});
  add_param(P, pre + ".norm2.weight", {C});
  add_param(P, pre + ".norm2.bias", {C});
  add_param(P, pre + ".conv1.conv.weight", {C, C, 3, 3, 3});
  add_param(P, pre + ".conv2.conv.weight", {C, C, 3, 3, 3});
}

static std::string down_name(int i, int j) { return "down_layers." + std::to_string(i) + "." + std::to_string(j); }
static std::string up_name(int i, int j) { return "up_layers." + std::to_string(i) + "." + std::to_string(j); }
static std::string up_conv_name(int i) { return "up_samples." + std::to_string(i) + ".0.conv.weight"; }

// in MONAI's registration order
static void segresnet_param_spec(Plan& P) {
  const b200unet_net_desc& d = P.d;
  const int L = d.n_levels, F = d.base_width;
  std::vector<int> Wd;
  for (int i = 0; i < L; ++i) Wd.push_back(F << i);
  add_param(P, "convInit.conv.weight", {F, d.n_features, 3, 3, 3});
  for (int i = 0; i < L; ++i) {
    if (i > 0) add_param(P, down_name(i, 0) + ".conv.weight", {Wd[i], Wd[i - 1], 3, 3, 3});
    for (int b = 1; b <= d.encoder_blocks[i]; ++b) add_segres_block_params(P, down_name(i, b), Wd[i]);
  }
  for (int i = 0; i + 1 < L; ++i)
    for (int b = 0; b < d.decoder_blocks[i]; ++b) add_segres_block_params(P, up_name(i, b), Wd[L - 2 - i]);
  for (int i = 0; i + 1 < L; ++i) add_param(P, up_conv_name(i), {Wd[L - 2 - i], 2 * Wd[L - 2 - i], 1, 1, 1});
  add_param(P, "conv_final.0.weight", {F});
  add_param(P, "conv_final.0.bias", {F});
  add_param(P, "conv_final.2.conv.weight", {d.n_outputs, F, 1, 1, 1});
  add_param(P, "conv_final.2.conv.bias", {d.n_outputs});
}

static int build_segresnet(Plan& P) {
  const b200unet_net_desc& d = P.d;
  const int L = d.n_levels, N = d.batch, F = d.base_width;
  B200_REQUIRE(L >= 2 && L <= 8, E_UNSUPPORTED, "plan: SegResNet with %d levels unsupported (2..8)", L);
  B200_REQUIRE(F >= 8 && F % 8 == 0, E_UNSUPPORTED, "plan: init_filters=%d must be a positive multiple of 8", F);
  B200_REQUIRE(F << (L - 1) <= 1024, E_UNSUPPORTED, "plan: SegResNet widths up to %d channels unsupported (the norms take at most 1024)",
               F << (L - 1));
  B200_REQUIRE(d.norm_groups >= 1 && F % d.norm_groups == 0, E_UNSUPPORTED, "plan: num_groups=%d must divide init_filters=%d",
               d.norm_groups, F);
  B200_REQUIRE(d.n_features >= 1 && d.n_features <= 16, E_UNSUPPORTED, "plan: in_channels=%d unsupported", d.n_features);
  B200_REQUIRE(d.n_outputs >= 1 && d.n_outputs <= B200_HEAD_MAX_OUTPUTS, E_UNSUPPORTED, "plan: out_channels=%d unsupported (1..%d)",
               d.n_outputs, B200_HEAD_MAX_OUTPUTS);
  for (int i = 0; i < L; ++i)
    B200_REQUIRE(d.encoder_blocks[i] >= 1, E_UNSUPPORTED, "plan: blocks_down[%d]=%d must be at least 1", i, d.encoder_blocks[i]);
  for (int i = 0; i + 1 < L; ++i)
    B200_REQUIRE(d.decoder_blocks[i] >= 1, E_UNSUPPORTED, "plan: blocks_up[%d]=%d must be at least 1", i, d.decoder_blocks[i]);
  std::vector<int> Wd, Ds, Hs, Ws;
  for (int i = 0; i < L; ++i) Wd.push_back(F << i);
  B200_TRY(level_extents(d, Ds, Hs, Ws));
  segresnet_param_spec(P);

  // ---- forward
  const TRef in = emit_prologue(P, /*with_input_stats=*/false);
  // convInit, Dropout3d through the epilogue's per-(n, c) scale; the statistics are those of the scaled output
  const int cinit = new_conv(P, "convInit.conv.weight", F, d.n_features, 3, 1, P.input_grad);
  TRef X = full(P, new_buf(P, N, Ds[0], Hs[0], Ws[0], F));
  emit_conv_fwd(P, cinit, in, -1, kNone, kNone, X, true, /*scale=*/true);
  release_buf(P, in.buf);
  std::vector<std::vector<BlockRec>> enc(L), dec(L);
  std::vector<int> pre(L, -1);
  std::vector<TRef> down_x(L);
  for (int i = 0; i < L; ++i) {
    if (i > 0) {   // stride-2 convolution of the previous level's output, which stays live as the skip
      pre[i] = new_conv(P, down_name(i, 0) + ".conv.weight", Wd[i], Wd[i - 1], 3, 2, true);
      TRef Y = full(P, new_buf(P, N, Ds[i], Hs[i], Ws[i], Wd[i]));
      emit_conv_fwd(P, pre[i], X, -1, kNone, kNone, Y, true, false);
      X = Y;
    }
    const int nb = d.encoder_blocks[i];
    for (int b = 0; b < nb; ++b) {
      // the level output feeds a convolution, not a norm: no statistics
      TRef dest = full(P, new_buf(P, N, Ds[i], Hs[i], Ws[i], Wd[i]));
      enc[i].push_back(build_block_fwd(P, segres_block_keys(down_name(i, b + 1)), X, Wd[i], Wd[i], dest, /*want_stats=*/b + 1 < nb,
                                       false, false, /*scale_in=*/i == 0 && b == 0, /*x_dead=*/true));
      X = dest;
    }
    down_x[i] = X;
  }
  std::vector<int> upc(L, -1);
  std::vector<TRef> up_in(L), up_p(L), up_y(L);
  for (int i = 0; i + 1 < L; ++i) {
    const int j = L - 2 - i, C = Wd[j];
    upc[i] = new_conv(P, up_conv_name(i), C, 2 * C, 1, 1, true);
    up_in[i] = X;
    up_p[i] = full(P, new_buf(P, N, Ds[j + 1], Hs[j + 1], Ws[j + 1], C));
    emit_conv_fwd(P, upc[i], X, -1, kNone, kNone, up_p[i], false, false);
    release_if_whole(P, X);
    up_y[i] = full(P, new_buf(P, N, Ds[j], Hs[j], Ws[j], C));
    emit_upsample2x_fwd(P, up_p[i], up_y[i], down_x[j]);
    release_buf(P, up_p[i].buf);
    release_if_whole(P, down_x[j]);
    X = up_y[i];
    const int nb = d.decoder_blocks[i];
    for (int b = 0; b < nb; ++b) {
      // the last stage's output feeds the head's GroupNorm; the other stages' feed a 1x1x1 convolution
      TRef dest = full(P, new_buf(P, N, Ds[j], Hs[j], Ws[j], C));
      dec[i].push_back(build_block_fwd(P, segres_block_keys(up_name(i, b)), X, C, C, dest, /*want_stats=*/b + 1 < nb || j == 0,
                                       false, false, false, /*x_dead=*/true));
      X = dest;
    }
  }
  // head: GroupNorm + act into a buffer, then the biased 1x1x1 head
  const int nf = new_norm(P, "conv_final.0", F, F, (long long)Ds[0] * Hs[0] * Ws[0], groups_for(F, d.norm_groups));
  const TRef A = full(P, new_buf(P, N, Ds[0], Hs[0], Ws[0], F));
  emit_norm_fwd(P, nf, X, A);
  release_if_whole(P, X);
  TRef g;
  B200_TRY(emit_head(P, A, P.find_param("conv_final.2.conv.weight"), P.find_param("conv_final.2.conv.bias"), &g));
  if (P.infer) return finish_build(P);

  // ---- backward
  g = emit_act_norm_bwd(P, nf, X, g, kNone);
  std::vector<TRef> dskip(L, kNone);
  for (int i = L - 2; i >= 0; --i) {   // up stages, top to bottom
    const int j = L - 2 - i, C = Wd[j];
    for (int b = d.decoder_blocks[i] - 1; b >= 0; --b) g = build_block_bwd(P, dec[i][b], g);
    // d(up(p) + skip): unchanged to the skip, through the adjoint of the up-sampling to the 1x1x1 convolution
    dskip[j] = g;
    TRef dP = full(P, new_buf(P, N, Ds[j + 1], Hs[j + 1], Ws[j + 1], C));
    emit_upsample2x_bwd(P, g, dP);
    emit_wgrad(P, upc[i], up_in[i], dP);
    TRef gX = full(P, new_buf(P, N, Ds[j + 1], Hs[j + 1], Ws[j + 1], 2 * C));
    emit_dgrad(P, upc[i], dP, gX, -1, kNone, kNone, false);
    g = gX;
  }
  // g = gradient of the bottom level's output; encoder, bottom to top
  for (int i = L - 1; i >= 0; --i) {
    for (int b = d.encoder_blocks[i] - 1; b >= 0; --b) g = build_block_bwd(P, enc[i][b], g);
    if (i > 0) g = emit_down_bwd(P, pre[i], down_x[i - 1], g, dskip[i - 1], false);
  }
  // g = gradient of convInit's output (the first ResBlock applied the dropout scale to it)
  emit_wgrad(P, cinit, in, g);
  if (P.input_grad) emit_input_dgrad(P, cinit, g, in, -1, kNone);
  emit_unpack_wgrads(P);
  return finish_build(P);
}

static int build(Plan& P) { return P.d.arch == 2 ? build_segresnet(P) : P.d.arch == 1 ? build_dynunet(P) : build_unet3d(P); }

// runs ops [first, last) of a schedule.  B200UNET_CAPTURE_DEBUG=1: after every op, check whether it invalidated an ongoing
// CUDA-graph capture of the stream, and name it if so.
static int run_ops(Plan& P, const std::vector<OpFn>& list, size_t first, size_t last, RunCtx& cx, const char* who) {
  static const bool capdbg = getenv("B200UNET_CAPTURE_DEBUG") != nullptr;
  for (size_t i = first; i < last; ++i) {
    int s = list[i](cx);
    if (s != OK) return s;
    if (capdbg) {
      cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
      cudaError_t e = cudaStreamIsCapturing(cx.st, &cs);
      if (e != cudaSuccess || cs == cudaStreamCaptureStatusInvalidated) {
        set_error("%s: stream capture invalidated at op '%s' (%s)", who, cx.label ? cx.label : "?", cudaGetErrorString(e));
        cudaGetLastError();
        return E_CUDA;
      }
    }
  }
  P.last_launches = cx.launches;
  return OK;
}

}  // namespace b200

extern "C" {

int b200unet_plan_create(const b200unet_net_desc* desc, b200unet_plan** out) {
  if (!desc || !out) { set_error("plan_create: null argument"); return E_INVALID; }
  b200unet_plan* P = new b200unet_plan();
  P->d = *desc;
  P->split = desc->split_precision != 0;
  P->infer = desc->inference_only != 0;
  P->deterministic = desc->deterministic != 0;
  P->input_grad = desc->input_grad != 0;
  P->slope = desc->act_slope;
  if (P->input_grad && P->infer) {
    set_error("plan_create: input_grad=1 on an inference_only plan (the input gradient needs the backward schedule)");
    delete P;
    *out = nullptr;
    return E_INVALID;
  }
  if (P->d.norm_groups <= 0) P->d.norm_groups = 8;
  if (P->d.feature_dilation <= 0) P->d.feature_dilation = 2;
  int s = build(*P);
  if (s != OK) { delete P; *out = nullptr; return s; }
  *out = P;
  return OK;
}

void b200unet_plan_destroy(b200unet_plan* plan) { delete plan; }

int b200unet_plan_num_params(const b200unet_plan* plan) { return plan ? (int)plan->params.size() : 0; }

int b200unet_plan_param_info(const b200unet_plan* plan, int i, int64_t shape[5], char* key, int key_cap) {
  if (!plan || i < 0 || i >= (int)plan->params.size()) { set_error("param_info: index out of range"); return E_INVALID; }
  const ParamInfo& p = plan->params[i];
  for (int k = 0; k < 5; ++k) shape[k] = p.shape[k];
  if (key && key_cap > 0) { strncpy(key, p.key.c_str(), key_cap - 1); key[key_cap - 1] = 0; }
  return p.ndim;
}

size_t b200unet_plan_workspace_bytes(const b200unet_plan* plan) { return plan ? plan->cur + 1024 : 0; }

int b200unet_plan_forward(b200unet_plan* plan, const float* x, const float* const* params, const float* dropout_scale,
                          int save_for_backward, void* workspace, float* logits, void* stream) {
  // save_for_backward: bit 0 = b200unet_plan_backward will follow; bit 1 = the parameters are unchanged since the previous
  // forward on THIS workspace: keep its packed bf16 weights (tiled inference runs 9-27 forwards per volume on fixed weights)
  const bool skip_pack = (save_for_backward & 2) != 0;
  save_for_backward &= 1;
  if (save_for_backward && plan && plan->infer) {
    set_error("plan_forward: save_for_backward=1 on a plan created with inference_only=1");
    return E_INVALID;
  }
  if (!plan || !x || !params || !workspace || !logits) { set_error("plan_forward: null argument"); return E_INVALID; }
  RunCtx cx(workspace, stream, plan->prof);
  cx.params = params; cx.x = x; cx.logits = logits;
  cx.skip_pack = skip_pack && plan->jobs_uploaded_for == cx.ws;   // only valid on a workspace that has been packed before
  plan->have_drop = dropout_scale != nullptr;
  if (dropout_scale) {
    float* dst = reinterpret_cast<float*>(cx.ws + plan->drop_off);
    if (cudaMemcpyAsync(dst, dropout_scale, sizeof(float) * plan->d.batch * plan->d.base_width, cudaMemcpyDeviceToDevice,
                        cx.st) != cudaSuccess) { set_error("plan_forward: dropout copy failed"); return E_CUDA; }
    cx.drop = dst;
  }
  return run_ops(*plan, plan->fwd, 0, plan->fwd.size(), cx, "plan_forward");
}

int b200unet_plan_backward(b200unet_plan* plan, const float* dlogits, const float* const* params, float* const* grads,
                           void* workspace, void* stream) {
  if (!plan || !dlogits || !params || !grads || !workspace) { set_error("plan_backward: null argument"); return E_INVALID; }
  if (plan->infer) { set_error("plan_backward: this plan was created with inference_only=1 (no backward schedule)"); return E_INVALID; }
  RunCtx cx(workspace, stream, plan->prof);
  cx.params = params; cx.grads = grads; cx.dlogits = dlogits;
  if (plan->have_drop) cx.drop = reinterpret_cast<float*>(cx.ws + plan->drop_off);
  return run_ops(*plan, plan->bwd, 0, plan->bwd.size(), cx, "plan_backward");
}

int b200unet_plan_input_grad(b200unet_plan* plan, float* dx, void* workspace, void* stream) {
  if (!plan || !dx || !workspace) { set_error("plan_input_grad: null argument"); return E_INVALID; }
  if (!plan->input_grad) { set_error("plan_input_grad: this plan was created without input_grad=1"); return E_INVALID; }
  RunCtx cx(workspace, stream, plan->prof);
  cx.dx = dx;
  return run_ops(*plan, plan->igrad, 0, plan->igrad.size(), cx, "plan_input_grad");
}

int b200unet_plan_last_launches(const b200unet_plan* plan) { return plan ? plan->last_launches : 0; }

int b200unet_plan_algorithmic_macs(const b200unet_plan* plan, double* macs, int ncat) {
  if (!plan || !macs) { set_error("algorithmic_macs: null argument"); return E_INVALID; }
  for (int i = 0; i < ncat; ++i) macs[i] = i < CAT_COUNT ? plan->macs[i] : 0.0;
  return OK;
}

int b200unet_plan_profile_begin(b200unet_plan* plan, int max_launches) {
  if (!plan || max_launches <= 0) { set_error("profile_begin: bad argument"); return E_INVALID; }
  if (plan->prof) { set_error("profile_begin: already profiling"); return E_INVALID; }
  Prof* p = new Prof();
  p->ev.resize((size_t)max_launches * 2);
  p->cat.resize(max_launches);
  p->label.resize(max_launches);
  for (auto& e : p->ev)
    if (cudaEventCreate(&e) != cudaSuccess) { set_error("profile_begin: cudaEventCreate failed"); delete p; return E_CUDA; }
  plan->prof = p;
  return OK;
}

int b200unet_plan_profile_dump(b200unet_plan* plan, const char* path) {
  if (!plan || !plan->prof || !path) { set_error("profile_dump: not profiling"); return E_INVALID; }
  Prof* p = plan->prof;
  FILE* f = fopen(path, "w");
  if (!f) { set_error("profile_dump: cannot open %s", path); return E_INVALID; }
  fprintf(f, "idx,category,ms,label\n");
  for (size_t i = 0; i < p->used; ++i) {
    if (cudaEventSynchronize(p->ev[i * 2 + 1]) != cudaSuccess) break;
    float ms = 0.f;
    cudaEventElapsedTime(&ms, p->ev[i * 2], p->ev[i * 2 + 1]);
    fprintf(f, "%zu,%d,%.6f,%s\n", i, p->cat[i], ms, p->label[i].c_str());
  }
  fclose(f);
  return OK;
}

int b200unet_plan_profile_end(b200unet_plan* plan, double* ms_by_cat, int64_t* launches_by_cat, int ncat) {
  if (!plan || !plan->prof || !ms_by_cat || !launches_by_cat) { set_error("profile_end: not profiling"); return E_INVALID; }
  Prof* p = plan->prof;
  plan->prof = nullptr;
  for (int i = 0; i < ncat; ++i) { ms_by_cat[i] = 0; launches_by_cat[i] = 0; }
  int status = p->overflow ? E_INVALID : OK;
  if (p->overflow) set_error("profile_end: event pool too small");
  for (size_t i = 0; i < p->used; ++i) {
    if (cudaEventSynchronize(p->ev[i * 2 + 1]) != cudaSuccess) { status = E_CUDA; set_error("profile_end: event sync failed"); break; }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, p->ev[i * 2], p->ev[i * 2 + 1]);
    const int c = p->cat[i];
    if (c < ncat) { ms_by_cat[c] += ms; launches_by_cat[c] += 1; }
  }
  for (auto& e : p->ev) cudaEventDestroy(e);
  delete p;
  return status;
}

}  // extern "C"
