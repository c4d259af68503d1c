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
  int part = -1;                   // backward only: -1 = the whole schedule; 0 / 1 = the part b200unet_plan_backward_part runs
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

struct ConvLayer {
  int pw;                  // parameter index
  int Co, Ci, Cop, Cip, ksz, stride, T;
  size_t wf_hi, wf_lo;     // packed forward weights   [T][Cop][Cip]
  size_t wd_hi, wd_lo;     // packed data-grad weights [T][Cip][Cop]
  size_t dw;               // fp32 accumulator         [T][Cip][Cop]
  bool need_dgrad;
  bool transposed;         // nn.ConvTranspose3d weight [Ci][Co][T] (+ bias parameter pb)
  bool up2;                // ConvTranspose3d with kernel = stride = 2 (MONAI UnetUpBlock): T = 8, weight [Ci][Co][8], no padding
  int pb;
  std::string name;        // state-dict key (profiling labels)
};

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
  std::vector<PackJob> pack_jobs, unpack_jobs;   // batched weight (un)packing tables (host copies)
  size_t jobs_off = 0;                           // device copy: pack jobs then unpack jobs
  const void* jobs_uploaded_for = nullptr;       // workspace base the table was last uploaded into
  Prof* prof = nullptr;
  double macs[CAT_COUNT] = {0, 0, 0, 0, 0, 0, 0, 0};  // algorithmic MACs per forward+backward pass, by category
  size_t drop_off = 0;      // [N][base_width] floats: copy of the dropout scale of the last forward
  bool have_drop = false;
  bool deterministic = false;   // weight gradients: per-split partial sums + fixed-order reduction instead of fp32 atomics
  size_t head_part_off = 0;   // per-block partial sums of the head weight gradient (fixed-order reduction)
  size_t wg_part_off = 0, wg_part_bytes = 0;   // scratch shared by all weight-gradient launches (stream-ordered)
  float slope = 0.f;        // negative slope of the activation (0 = ReLU: UNet3D; 0.01 = LeakyReLU: DynUNet)
  bool infer = false;       // forward-only plan: no backward schedule / buffers, forward temporaries are recycled
  // two-part backward (b200unet_plan_backward_part): part 0 = head, decoder and the deepest encoder level(s) -- most of the
  // parameters -- whose gradients can be exchanged between ranks while part 1 (the shallow encoder levels) still runs
  int bwd_split = -1;                 // index into bwd of the first op of part 1 (-1: one part)
  std::vector<int> param_last_op;     // per parameter: index of the last backward op that contributes to its gradient
  size_t unpack_split = 0;            // unpack jobs [0, unpack_split) belong to part 0
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

// the backward op about to be pushed contributes to the gradient of parameter `pidx`
static void touch(Plan& P, int pidx) {
  if (pidx < 0) return;
  if (P.param_last_op.size() < P.params.size()) P.param_last_op.resize(P.params.size(), -1);
  P.param_last_op[pidx] = (int)P.bwd.size();
}
static int param_part(const Plan& P, int pidx) {
  if (P.bwd_split < 0) return 0;
  if (pidx < 0 || pidx >= (int)P.param_last_op.size() || P.param_last_op[pidx] < 0) return 1;   // unknown writer: final only at the end
  return P.param_last_op[pidx] < P.bwd_split ? 0 : 1;
}

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

static void build_param_spec(Plan& P) {
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

static int new_conv(Plan& P, const std::string& key, int Co, int Ci, int ksz, int stride, bool need_dgrad) {
  ConvLayer c;
  c.pw = P.find_param(key);
  c.name = key;
  c.Co = Co; c.Ci = Ci; c.Cop = round_up(Co, 8); c.Cip = round_up(Ci, 8);
  c.ksz = ksz; c.stride = stride; c.T = ksz * ksz * ksz;
  need_dgrad = need_dgrad && !P.infer;
  c.need_dgrad = need_dgrad;
  c.transposed = false;
  c.up2 = false;
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

static int new_norm(Plan& P, const std::string& prefix, int C, int Cld, long long S) {
  NormLayer n;
  n.name = prefix;
  n.pg = P.find_param(prefix + ".weight");
  n.pb = P.find_param(prefix + ".bias");
  n.C = C; n.Cld = Cld; n.G = groups_for(C, P.d.norm_groups); n.S = S;
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

// A operand + packed weights of a convolution through layer c: its forward pack applied to x, or (dgrad) its data-gradient pack
// applied to x = the gradient of its output.  A convolution reads its input at its stride and its output gradient at stride 1
// (stride 2: parity-class mode); a transposed convolution reads its input at stride 1 (zero-inserted or parity-class mode) and
// its output gradient at stride 2.
static ConvSrc conv_src(const Plan& P, const RunCtx& cx, const ConvLayer& c, TRef x, bool dgrad) {
  const bool up = c.transposed || c.up2;
  ConvSrc s;
  memset(&s, 0, sizeof(s));
  s.x = act_of(P, cx, x);
  s.w_hi = reinterpret_cast<bf16*>(cx.ws + (dgrad ? c.wd_hi : c.wf_hi));
  s.w_lo = P.split ? reinterpret_cast<bf16*>(cx.ws + (dgrad ? c.wd_lo : c.wf_lo)) : nullptr;
  s.ksz = c.ksz;
  s.nopad = c.up2 ? 1 : 0;
  s.stride = up ? (dgrad ? 2 : 1) : (dgrad ? 1 : c.stride);
  s.Cip = dgrad ? c.Cop : c.Cip;   // K extent of the data-gradient pack [T][Cip][Cop] = Cop
  return s;
}

// generic forward-weights conv:  out = (conv(a, W[ci]) [+ conv1x1(a2, W[ci2])] [+ res]) [* dropout]
static double conv_macs(const Plan& P, int ci, TRef out_like) {
  const ConvLayer& c = P.convs[ci];
  const Buf& b = P.bufs[out_like.buf];
  return (double)b.N * b.D * b.H * b.W * c.Co * c.Ci * c.T / (c.transposed ? 8.0 : 1.0);
}

static void emit_conv_fwd(Plan& P, int ci, TRef a, int ci2, TRef a2, TRef res, TRef out, bool stats, bool scale) {
  if (stats) need_stats(P, out.buf);
  const int cat = CAT_CONV_FWD;
  P.macs[cat] += conv_macs(P, ci, out) + (ci2 >= 0 ? conv_macs(P, ci2, out) : 0.0);
  push_op(P.fwd, "conv_fwd " + P.convs[ci].name + " " + shape_of(P, a) + "->" + shape_of(P, out) + (ci2 >= 0 ? " +sample" : "") + (res.valid() ? " +res" : ""),
          [&P, ci, a, ci2, a2, res, out, stats, scale, cat](RunCtx& cx) -> int {
    const ConvLayer& c = P.convs[ci];
    ConvOp op;
    memset(&op, 0, sizeof(op));
    op.nsrc = 1;
    op.src[0] = conv_src(P, cx, c, a, false);
    op.Cop = c.Cop;
    if (ci2 >= 0) {
      op.nsrc = 2;
      op.src[1] = conv_src(P, cx, P.convs[ci2], a2, false);
    }
    op.out = act_of(P, cx, out);
    Act r;
    if (res.valid()) { r = act_of(P, cx, res); op.res = &r; }
    if (scale && cx.drop) op.scale = cx.drop;
    if (stats) { op.stats = stats_ptr(P, cx, out); op.stats_ld = P.bufs[out.buf].C; }
    if (c.transposed) { op.bias = cx.params[c.pb]; op.zero_last = 1; }
    LAUNCHED(cx, cat, launch_igemm_conv(op, cx.st));
    return OK;
  });
}

// ---- backward op emitters
static void size_wgrad_partials(Plan& P, const Act& a, const Act& dy, int ksz, int stride, int nopad, int Cip, int Cop) {
  if (!P.deterministic) return;
  WgradOp op;
  memset(&op, 0, sizeof(op));
  op.a = a; op.dy = dy; op.ksz = ksz; op.stride = stride; op.nopad = nopad; op.Cip = Cip; op.Cop = Cop;
  const size_t need = wgrad_partial_bytes(op, device_sms());
  if (need > P.wg_part_bytes) P.wg_part_bytes = need;
}

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

static void emit_wgrad(Plan& P, int ci, TRef a, TRef dy) {
  P.macs[CAT_CONV_WGRAD] += conv_macs(P, ci, dy);
  size_wgrad_partials(P, shape_act(P, a), shape_act(P, dy), P.convs[ci].ksz, P.convs[ci].stride, 0, P.convs[ci].Cip, P.convs[ci].Cop);
  touch(P, P.convs[ci].pw);
  push_op(P.bwd, "wgrad " + P.convs[ci].name + " " + shape_of(P, a) + " x " + shape_of(P, dy), [&P, ci, a, dy](RunCtx& cx) -> int {
    const ConvLayer& c = P.convs[ci];
    WgradOp op;
  memset(&op, 0, sizeof(op));
    op.a = act_of(P, cx, a);
    op.dy = act_of(P, cx, dy);
    op.ksz = c.ksz; op.stride = c.stride; op.nopad = 0; op.Cip = c.Cip; op.Cop = c.Cop;
    op.dw = reinterpret_cast<float*>(cx.ws + P.bz_off + c.dw);
    return run_wgrad(P, cx, op);
  });
}

// data gradient through conv `ci` (stride 1):  out = conv(dy, Wd)  with either the GN/ReLU backward epilogue
// (ni >= 0, gn_x = raw input of the norm) or a plain epilogue (+res, *dropout scale).
static void emit_dgrad(Plan& P, int ci, TRef dy, TRef out, int ni, TRef gn_x, TRef res, bool scale, double alg_macs,
                       bool cls_mode = false, std::vector<OpFn>* list = nullptr) {
  const int cat = CAT_CONV_DGRAD;
  P.macs[cat] += alg_macs;
  push_op(list ? *list : P.bwd, std::string(ni >= 0 ? "dgrad+gnrelu " : "dgrad ") + P.convs[ci].name + " " + shape_of(P, dy) + "->" + shape_of(P, out),
          [&P, ci, dy, out, ni, gn_x, res, scale, cat, cls_mode](RunCtx& cx) -> int {
    const ConvLayer& c = P.convs[ci];
    ConvOp op;
    memset(&op, 0, sizeof(op));
    op.nsrc = 1;
    op.cls_mode = cls_mode ? 1 : 0;
    op.src[0] = conv_src(P, cx, c, dy, true);
    op.Cop = c.Cip;   // rows of Wd = Cip
    op.out = act_of(P, cx, out);
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
  touch(P, P.norms[ni].pg);
  touch(P, P.norms[ni].pb);
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
  touch(P, P.norms[ni].pg);
  touch(P, P.norms[ni].pb);
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

// the per-parameter pointers (cx.params or cx.grads) as the batched (un)packing kernels take them
static PtrTable ptr_table(const Plan& P, const float* const* p) {
  PtrTable tbl;
  memset(&tbl, 0, sizeof(tbl));
  for (size_t i = 0; i < P.params.size(); ++i) tbl.p[i] = p[i];
  return tbl;
}

// First op of every forward: zero the statistics arena, upload the job tables into a new workspace, pack all weights (one
// launch) and pack the network input (with_input_stats: and its channel statistics, for a GroupNorm that reads it).
static void emit_prologue(Plan& P, int b_in, bool with_input_stats) {
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
}

// first op of every backward: zero the backward statistics and the weight-gradient accumulators
static void emit_bwd_memset(Plan& P) {
  push_op(P.bwd, "memset", [&P](RunCtx& cx) -> int {
    B200_CHECK_CUDA(cudaMemsetAsync(cx.ws + P.bz_off, 0, P.bz_bytes, cx.st));
    return OK;
  });
}

// The 1x1x1 head (bias_param >= 0: with a bias).  Training plans also get its backward op; returns the gradient of Xfinal
// (kNone in a forward-only plan).  launch_head_fwd / launch_head_bwd pick the kernels from n_outputs; above 8 outputs the
// bias gradient comes out of the same backward pass instead of launch_head_dbias.
static TRef emit_head(Plan& P, TRef Xfinal, int w_param, int bias_param) {
  P.head_param = w_param;
  push_op(P.fwd, "head_fwd", [&P, Xfinal, bias_param](RunCtx& cx) -> int {
    LAUNCHED(cx, CAT_HEAD, launch_head_fwd(act_of(P, cx, Xfinal), cx.params[P.head_param], P.d.n_outputs, P.d.activation, cx.logits, cx.st,
                                           bias_param >= 0 ? cx.params[bias_param] : nullptr));
    return OK;
  });
  if (P.infer) return kNone;
  const Buf xb = P.bufs[Xfinal.buf];
  const TRef g = full(P, new_buf(P, xb.N, xb.D, xb.H, xb.W, Xfinal.c));
  touch(P, w_param);
  touch(P, bias_param);
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
  return g;
}

// Everything pushed so far is part 0 of a two-part backward.  The op pushed here unpacks the weight gradients of part 0
// (accumulator -> torch layout) and runs only under b200unet_plan_backward_part(part = 0): the whole-schedule call unpacks
// every job in its last op (emit_unpack_wgrads).
static void emit_bwd_split(Plan& P) {
  push_op(P.bwd, "unpack_wgrads (part 0)", [&P](RunCtx& cx) -> int {
    if (cx.part != 0 || P.unpack_split == 0) return OK;
    const PackJob* jobs = reinterpret_cast<const PackJob*>(cx.ws + P.jobs_off) + P.pack_jobs.size();
    LAUNCHED(cx, CAT_PACK, launch_unpack_all(ptr_table(P, cx.grads), jobs, (int)P.unpack_split, cx.ws, cx.st));
    return OK;
  });
  P.bwd_split = (int)P.bwd.size();
}

// last op of every backward: weight gradients, accumulator -> torch layout (one batched launch)
static void emit_unpack_wgrads(Plan& P) {
  push_op(P.bwd, "unpack_wgrads", [&P](RunCtx& cx) -> int {
    // run as part 1 of a two-part backward, the jobs of part 0 were unpacked at the split (emit_bwd_split)
    const size_t first = cx.part == 1 ? P.unpack_split : 0;
    const PackJob* jobs = reinterpret_cast<const PackJob*>(cx.ws + P.jobs_off) + P.pack_jobs.size() + first;
    LAUNCHED(cx, CAT_PACK, launch_unpack_all(ptr_table(P, cx.grads), jobs, (int)(P.unpack_jobs.size() - first), cx.ws, cx.st));
    return OK;
  });
}

// ------------------------------------------------------------------------------------------------ residual block
static BlockRec build_block_fwd(Plan& P, const std::string& pre, TRef X, int cin_real, int C, TRef dest, bool want_stats,
                                bool first, bool scale_out, bool scale_in, bool x_dead) {
  const Buf& xb = P.bufs[X.buf];
  const int N = xb.N, D = xb.D, H = xb.H, W = xb.W;
  const long long S = (long long)D * H * W;
  BlockRec r;
  r.X = X; r.first = first; r.scale_out = scale_out; r.scale_in = scale_in;
  r.n1 = new_norm(P, pre + ".conv1.norm1", cin_real, X.c, S);
  r.c1 = new_conv(P, pre + ".conv1.conv.weight", C, cin_real, 3, 1, true);
  r.n2 = new_norm(P, pre + ".conv2.norm1", C, C, S);
  r.c2 = new_conv(P, pre + ".conv2.conv.weight", C, C, 3, 1, true);
  r.cs = (cin_real != C) ? new_conv(P, pre + ".sample.weight", C, cin_real, 1, 1, !first || P.input_grad) : -1;
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

// returns the TRef of dX (kNone for the first block of the network)
static TRef build_block_bwd(Plan& P, const BlockRec& r, TRef dOut) {
  const Buf& xb = P.bufs[r.X.buf];
  const int N = xb.N, D = xb.D, H = xb.H, W = xb.W;
  const int C = r.y1.c;
  emit_wgrad(P, r.c2, r.a2, dOut);
  if (r.cs >= 0) emit_wgrad(P, r.cs, r.X, dOut);
  TRef dz2 = full(P, new_buf(P, N, D, H, W, C));
  emit_dgrad(P, r.c2, dOut, dz2, r.n2, r.y1, kNone, false, conv_macs(P, r.c2, dOut));
  TRef dy1 = full(P, new_buf(P, N, D, H, W, C));
  emit_gn_bwd(P, r.n2, dz2, r.y1, kNone, dy1, false);
  emit_wgrad(P, r.c1, r.a1, dy1);
  TRef dz1 = full(P, new_buf(P, N, D, H, W, r.X.c));
  emit_dgrad(P, r.c1, dy1, dz1, r.n1, r.X, kNone, false, r.first ? 0.0 : conv_macs(P, r.c1, dy1));
  if (r.first) {   // no data gradient below the first block: only dgamma / dbeta of its first norm are needed
    emit_gn_bwd_finalize(P, r.n1);
    if (P.input_grad) {
      // dOut already carries the Dropout3d scale of this block's output (applied by whoever produced it): not applied again
      TRef res = dOut;
      if (r.cs >= 0) {
        res = full(P, new_buf(P, N, D, H, W, r.X.c));
        emit_dgrad(P, r.cs, dOut, res, -1, kNone, kNone, false, 0.0, false, &P.igrad);
      }
      emit_input_grad(P, r.n1, dz1, r.X, res);
    }
    return kNone;
  }
  TRef dX = full(P, new_buf(P, N, D, H, W, r.X.c));
  if (r.cs >= 0) {
    emit_gn_bwd(P, r.n1, dz1, r.X, kNone, dX, false);
    emit_dgrad(P, r.cs, dOut, dX, -1, kNone, dX, r.scale_in, conv_macs(P, r.cs, dOut));  // dX = (conv1x1(dOut, Ws^T) + dX) [* scale]
  } else {
    emit_gn_bwd(P, r.n1, dz1, r.X, dOut, dX, r.scale_in);
  }
  return dX;
}

static int finish_build(Plan& P);

static int build_unet3d(Plan& P) {
  const b200unet_net_desc& d = P.d;
  const int L = d.n_levels, N = d.batch;
  B200_REQUIRE(L >= 2 && L <= 8, E_UNSUPPORTED, "plan: n_levels=%d unsupported (2..8)", L);
  B200_REQUIRE(d.base_width % 8 == 0, E_UNSUPPORTED, "plan: base_width=%d must be a multiple of 8", d.base_width);
  B200_REQUIRE(d.n_features >= 1 && d.n_features <= 16, E_UNSUPPORTED, "plan: n_features=%d unsupported", d.n_features);
  B200_REQUIRE(d.n_outputs >= 1 && d.n_outputs <= B200_HEAD_MAX_OUTPUTS, E_UNSUPPORTED, "plan: n_outputs=%d unsupported (1..%d)",
               d.n_outputs, B200_HEAD_MAX_OUTPUTS);
  std::vector<int> widths, Ds, Hs, Ws;
  {
    int w = d.base_width, D = d.depth, H = d.height, W = d.width;
    for (int li = 0; li < L; ++li) {
      widths.push_back(w); Ds.push_back(D); Hs.push_back(H); Ws.push_back(W);
      if (li + 1 < L)
        B200_REQUIRE(D % 2 == 0 && H % 2 == 0 && W % 2 == 0 && D >= 2 && H >= 2 && W >= 2, E_UNSUPPORTED,
                     "plan: level %d extent %dx%dx%d must be even (input %dx%dx%d not divisible by 2^%d)", li, D, H, W,
                     d.depth, d.height, d.width, L - 1);
      w *= d.feature_dilation; D /= 2; H /= 2; W /= 2;
    }
  }
  build_param_spec(P);

  // ---------------- forward
  const int Cp_in = round_up(d.n_features, 8);
  const int b_in = new_buf(P, N, Ds[0], Hs[0], Ws[0], Cp_in);
  emit_prologue(P, b_in, /*with_input_stats=*/true);

  std::vector<std::vector<BlockRec>> enc(L), dec(L);
  std::vector<int> cat(L, -1), down(L, -1);
  std::vector<TRef> skip(L), down_out(L);
  std::vector<StageRec> stages;
  for (int li = 0; li + 1 < L; ++li) {
    cat[li] = new_buf(P, N, Ds[li], Hs[li], Ws[li], 2 * widths[li]);
    need_stats(P, cat[li]);
  }
  TRef X = full(P, b_in);
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
      enc[li].push_back(build_block_fwd(P, "encoder.layers." + std::to_string(li) + ".blocks." + std::to_string(b), X,
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
      dec[i].push_back(build_block_fwd(P, "decoder.layers." + std::to_string(i) + ".blocks." + std::to_string(b), X, in_w,
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
      TRef Pin = s.P, U = s.U;
      push_op(P.fwd, "upsample2x_fwd " + shape_of(P, Pin), [&P, Pin, U](RunCtx& cx) -> int {
        LAUNCHED(cx, CAT_RESAMPLE, launch_upsample2x_fwd(act_of(P, cx, Pin), act_of(P, cx, U), stats_ptr(P, cx, U), P.bufs[U.buf].C,
                                           cx.st));
        return OK;
      });
      release_buf(P, s.P.buf);
    } else {
      // ConvTranspose3d(k3, s2, p1) + bias, then F.pad(+1 high side) = zero-insert + 3x3x3 conv with the flipped
      // kernel over a 2n grid whose last plane/row/column is forced to 0 (decoder.py:101-102, unet.py:34-40)
      const std::string key = "decoder.upsampling_blocks." + std::to_string(i);
      s.cup = new_conv(P, key + ".weight", out_w, in_w, 3, 1, true);
      P.convs[s.cup].transposed = true;
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
      dec[L - 1].push_back(build_block_fwd(P, "decoder.layers." + std::to_string(L - 1) + ".blocks." + std::to_string(b), X,
                                           cin, d.base_width, dest, b + 1 < d.decoder_blocks[L - 1], false, false, false, true));
      X = dest;
      cin = d.base_width;
    }
  }
  if (!P.infer) {
    B200_REQUIRE(d.activation == 0, E_UNSUPPORTED,
                 "plan: activation inside the model (sigmoid/softmax) is inference-only; train on logits");
    emit_bwd_memset(P);
  }
  TRef g = emit_head(P, X, P.find_param("final_convolution.weight"), -1);

  // ---------------- backward (training plans only)
  if (!P.infer) {
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
      push_op(P.bwd, "upsample2x_bwd " + shape_of(P, dP), [&P, dU, dP](RunCtx& cx) -> int {
        LAUNCHED(cx, CAT_RESAMPLE, launch_upsample2x_bwd(act_of(P, cx, dU), act_of(P, cx, dP), cx.st));
        return OK;
      });
      emit_wgrad(P, s.cpre, s.Xin, dP);
      emit_dgrad(P, s.cpre, dP, gX, -1, kNone, kNone, false, conv_macs(P, s.cpre, dP));
    } else {
      // the padded boundary of the ConvT output is a constant: mask it out of dU (visible extent 2n-1 through TMA)
      TRef dUm = masked(dU);
      const int cup = s.cup;
      touch(P, P.convs[cup].pb);
      push_op(P.bwd, "bias_grad " + P.convs[cup].name, [&P, dUm, cup](RunCtx& cx) -> int {
        LAUNCHED(cx, CAT_OTHER, launch_bias_grad(act_of(P, cx, dUm), cx.grads[P.convs[cup].pb], cx.st));
        return OK;
      });
      emit_wgrad(P, cup, s.Z, dUm);                                   // dW[tap][ci][co] from the zero-inserted input
      emit_dgrad(P, cup, dUm, gX, -1, kNone, kNone, false, conv_macs(P, cup, dUm));   // stride-2 conv of dU: dX[i] = sum_k dU[2i+k-1] W[ci][co][k]
    }
    for (int b = d.decoder_blocks[i] - 1; b >= 0; --b) gX = build_block_bwd(P, dec[i][b], gX);
    g = gX;
  }
  // g = gradient w.r.t. the bottleneck output (skip[L-1])
  for (int li = L - 1; li >= 0; --li) {
    for (int b = d.encoder_blocks[li] - 1; b >= 0; --b) g = build_block_bwd(P, enc[li][b], g);
    if (li > 0) {
      const int lj = li - 1;
      emit_wgrad(P, down[lj], skip[lj], g);
      // head, decoder and the deepest encoder level are done: ~90 % of the parameters (C2: 21.4 M of 24.0 M) have their
      // gradients, ~25 % of the backward time is still ahead
      if (li == L - 1) emit_bwd_split(P);
      TRef gin = g;
      TRef gS = full(P, new_buf(P, N, Ds[lj], Hs[lj], Ws[lj], widths[lj]));
      // dropout scale belongs to the output of encoder block (0,0): that is this tensor iff level 0 has one block
      const bool sc = (lj == 0 && d.encoder_blocks[0] == 1);
      // eight parity-class implicit GEMMs over the un-inserted gradient (27 tap products instead of 8 x 27), TMA-stored
      // into their interleaved positions
      emit_dgrad(P, down[lj], gin, gS, -1, kNone, dskip_dec[lj], sc, conv_macs(P, down[lj], gin), /*cls_mode=*/true);
      g = gS;
    }
  }
  emit_unpack_wgrads(P);
  }  // !P.infer
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
  const int head_c = d.arch == 1 ? d.filters[0] : d.base_width;
  B200_REQUIRE(d.n_outputs <= 8 || head_c <= 64, E_UNSUPPORTED,
               "plan: more than 8 outputs need at most 64 channels into the head, got %d", head_c);
  if (!P.infer) P.head_part_off = P.alloc(head_bwd_scratch_bytes(d.n_outputs, head_c));
  for (size_t i = 0; i < P.convs.size(); ++i)
    B200_REQUIRE(P.convs[i].pw >= 0, E_INVALID, "plan: internal: conv %d has no parameter", (int)i);
  for (const ConvLayer& c : P.convs) {
    PackJob j;
    j.pidx = c.pw; j.Co = c.Co; j.Ci = c.Ci; j.Cop = c.Cop; j.Cip = c.Cip; j.T = c.T;
    j.mode = c.up2 ? 4 : c.transposed ? 2 : 0; j.off_hi = (long long)c.wf_hi; j.off_lo = (long long)c.wf_lo;
    P.pack_jobs.push_back(j);
    if (c.need_dgrad) {
      j.mode = (c.up2 || c.transposed) ? 3 : 1; j.off_hi = (long long)c.wd_hi; j.off_lo = (long long)c.wd_lo;
      P.pack_jobs.push_back(j);
    }
    if (P.infer) continue;
    PackJob u = j;
    u.mode = c.transposed ? 2 : 0; u.off_hi = (long long)(P.bz_off + c.dw); u.off_lo = 0;
    if (c.up2) {   // accumulated with swapped roles as [T][pad(Co)][pad(Ci)] (see emit_wgrad_up2): reads back as [Ci][Co][T]
      u.mode = 0; u.Co = c.Ci; u.Ci = c.Co; u.Cop = c.Cip; u.Cip = c.Cop;
    }
    // the jobs of part 0 of a two-part backward first (b200unet_plan_backward_part), the others behind them
    if (param_part(P, c.pw) == 0 && P.bwd_split >= 0) P.unpack_jobs.insert(P.unpack_jobs.begin() + P.unpack_split++, u);
    else P.unpack_jobs.push_back(u);
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

static int new_norm_keys(Plan& P, const std::string& prefix, int C, long long S) {
  const int ni = new_norm(P, prefix, C, C, S);
  P.norms[ni].G = C;   // instance norm: one group per channel
  return ni;
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
  r.n1 = new_norm_keys(P, pre + ".norm1", C, S);
  r.n2 = new_norm_keys(P, pre + ".norm2", C, S);
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

static void emit_act_bwd(Plan& P, int ni, TRef g1, TRef g2, TRef c, TRef dz) {
  push_op(P.bwd, "act_bwd " + P.norms[ni].name + " " + shape_of(P, c), [&P, ni, g1, g2, c, dz](RunCtx& cx) -> int {
    const NormLayer& n = P.norms[ni];
    Act a2;
    if (g2.valid()) a2 = act_of(P, cx, g2);
    LAUNCHED(cx, CAT_NORM, launch_act_bwd(act_of(P, cx, g1), g2.valid() ? &a2 : nullptr, act_of(P, cx, c),
                                          reinterpret_cast<float*>(cx.ws + n.coef), P.slope, act_of(P, cx, dz),
                                          reinterpret_cast<double*>(cx.ws + P.bz_off + n.bstats), n.Cld, cx.st));
    return OK;
  });
}

// gradient of the block output arrives as g1 (+ g2); returns dX (kNone for the first block)
static TRef build_dyn_block_bwd(Plan& P, const DynBlock& r, TRef g1, TRef g2) {
  const Buf& cb = P.bufs[r.c1.buf];
  const int N = cb.N, D = cb.D, H = cb.H, W = cb.W, C = r.c1.c;
  TRef dz2 = full(P, new_buf(P, N, D, H, W, C));
  emit_act_bwd(P, r.n2, g1, g2, r.c2, dz2);
  TRef dc2 = full(P, new_buf(P, N, D, H, W, C));
  emit_gn_bwd(P, r.n2, dz2, r.c2, kNone, dc2, false);
  emit_wgrad(P, r.k2, r.a1, dc2);
  TRef dz1 = full(P, new_buf(P, N, D, H, W, C));
  emit_dgrad(P, r.k2, dc2, dz1, r.n1, r.c1, kNone, false, conv_macs(P, r.k2, dc2));   // mode 1: masked by act'(norm1(c1)) + statistics
  TRef dc1 = full(P, new_buf(P, N, D, H, W, C));
  emit_gn_bwd(P, r.n1, dz1, r.c1, kNone, dc1, false);
  emit_wgrad(P, r.k1, r.X, dc1);
  if (r.first) {
    if (P.input_grad) {
      const Buf& xb = P.bufs[r.X.buf];
      TRef dX = full(P, new_buf(P, N, xb.D, xb.H, xb.W, r.X.c));
      emit_dgrad(P, r.k1, dc1, dX, -1, kNone, kNone, false, 0.0, r.stride == 2, &P.igrad);
      emit_input_grad(P, -1, kNone, kNone, dX);
    }
    return kNone;
  }
  const Buf& xb = P.bufs[r.X.buf];
  TRef dX = full(P, new_buf(P, N, xb.D, xb.H, xb.W, r.X.c));
  emit_dgrad(P, r.k1, dc1, dX, -1, kNone, kNone, false, conv_macs(P, r.k1, dc1), /*cls_mode=*/r.stride == 2);
  return dX;
}

static int build_dynunet(Plan& P) {
  const b200unet_net_desc& d = P.d;
  const int L = d.n_levels, N = d.batch;
  B200_REQUIRE(L >= 2 && L <= 8, E_UNSUPPORTED, "plan: DynUNet with %d levels unsupported (2..8)", L);
  B200_REQUIRE(d.n_features >= 1 && d.n_features <= 16, E_UNSUPPORTED, "plan: in_channels=%d unsupported", d.n_features);
  B200_REQUIRE(d.n_outputs >= 1 && d.n_outputs <= B200_HEAD_MAX_OUTPUTS, E_UNSUPPORTED, "plan: out_channels=%d unsupported (1..%d)",
               d.n_outputs, B200_HEAD_MAX_OUTPUTS);
  P.slope = d.act_slope;
  std::vector<int> F, Ds, Hs, Ws;
  {
    int D = d.depth, H = d.height, W = d.width;
    for (int i = 0; i < L; ++i) {
      B200_REQUIRE(d.filters[i] >= 8 && d.filters[i] % 8 == 0, E_UNSUPPORTED, "plan: filters[%d]=%d must be a positive multiple of 8", i,
                   d.filters[i]);
      F.push_back(d.filters[i]); Ds.push_back(D); Hs.push_back(H); Ws.push_back(W);
      if (i + 1 < L)
        B200_REQUIRE(D % 2 == 0 && H % 2 == 0 && W % 2 == 0 && D >= 2 && H >= 2 && W >= 2, E_UNSUPPORTED,
                     "plan: level %d extent %dx%dx%d must be even (input %dx%dx%d not divisible by 2^%d)", i, D, H, W, d.depth,
                     d.height, d.width, L - 1);
      D /= 2; H /= 2; W /= 2;
    }
  }
  // ---- parameter spec in MONAI's registration order: input_block, downsamples, bottleneck, upsamples, output_block
  auto enc_name = [&](int i) -> std::string {
    return i == 0 ? "input_block" : i == L - 1 ? "bottleneck" : "downsamples." + std::to_string(i - 1);
  };
  for (int i = 0; i < L; ++i) add_dyn_block_params(P, enc_name(i), i == 0 ? d.n_features : F[i - 1], F[i]);
  for (int u = 0; u + 1 < L; ++u) {      // upsamples[u] maps level L-1-u -> L-2-u
    const int lo = L - 1 - u, hi = L - 2 - u;
    const std::string pre = "upsamples." + std::to_string(u);
    add_param(P, pre + ".transp_conv.conv.weight", {F[lo], F[hi], 2, 2, 2});
    add_dyn_block_params(P, pre + ".conv_block", 2 * F[hi], F[hi]);
  }
  add_param(P, "output_block.conv.conv.weight", {d.n_outputs, F[0], 1, 1, 1});
  add_param(P, "output_block.conv.conv.bias", {d.n_outputs});

  // ---- forward
  const int Cp_in = round_up(d.n_features, 8);
  const int b_in = new_buf(P, N, Ds[0], Hs[0], Ws[0], Cp_in);
  emit_prologue(P, b_in, /*with_input_stats=*/false);
  std::vector<int> cat(L, -1);
  for (int i = 0; i + 1 < L; ++i) cat[i] = new_buf(P, N, Ds[i], Hs[i], Ws[i], 2 * F[i]);
  std::vector<DynBlock> enc(L), dec(L);
  std::vector<int> up(L, -1);
  TRef X = full(P, b_in);
  int cin_real = d.n_features;
  for (int i = 0; i < L; ++i) {
    TRef dest = (i + 1 < L) ? slice(full(P, cat[i]), F[i], F[i]) : full(P, new_buf(P, N, Ds[i], Hs[i], Ws[i], F[i]));
    enc[i] = build_dyn_block_fwd(P, enc_name(i), X, cin_real, F[i], i == 0 ? 1 : 2, dest, i == 0, /*x_dead=*/i == 0);
    X = dest;
    cin_real = F[i];
  }
  for (int u = 0; u + 1 < L; ++u) {
    const int lo = L - 1 - u, hi = L - 2 - u;
    const std::string pre = "upsamples." + std::to_string(u);
    up[hi] = new_conv(P, pre + ".transp_conv.conv.weight", F[hi], F[lo], 2, 2, true);
    P.convs[up[hi]].up2 = true;
    TRef U = slice(full(P, cat[hi]), 0, F[hi]);
    {
      const int ci = up[hi];
      TRef Xin = X;
      P.macs[CAT_CONV_FWD] += (double)N * Ds[lo] * Hs[lo] * Ws[lo] * F[lo] * F[hi] * 8;
      push_op(P.fwd, "convT_k2s2 " + P.convs[ci].name + " " + shape_of(P, Xin) + "->" + shape_of(P, U), [&P, ci, Xin, U](RunCtx& cx) -> int {
        const ConvLayer& c = P.convs[ci];
        ConvOp op;
        memset(&op, 0, sizeof(op));
        op.nsrc = 1;
        op.cls_mode = 2;
        op.src[0] = conv_src(P, cx, c, Xin, false);
        op.Cop = c.Cop;
        op.out = act_of(P, cx, U);
        LAUNCHED(cx, CAT_CONV_FWD, launch_igemm_conv(op, cx.st));
        return OK;
      });
    }
    release_if_whole(P, X);
    TRef dest = full(P, new_buf(P, N, Ds[hi], Hs[hi], Ws[hi], F[hi]));
    dec[hi] = build_dyn_block_fwd(P, pre + ".conv_block", full(P, cat[hi]), 2 * F[hi], F[hi], 1, dest, false, /*x_dead=*/true);
    X = dest;
  }
  if (!P.infer) {
    B200_REQUIRE(d.activation == 0, E_UNSUPPORTED, "plan: activation inside the model is inference-only; train on logits");
    emit_bwd_memset(P);
  }
  TRef g = emit_head(P, X, P.find_param("output_block.conv.conv.weight"), P.find_param("output_block.conv.conv.bias"));
  if (P.infer) return finish_build(P);

  // ---- backward
  std::vector<TRef> dskip(L, kNone);
  for (int hi = 0; hi + 1 < L; ++hi) {     // decoder, top (level 0) to bottom
    const int lo = hi + 1;
    TRef dCat = build_dyn_block_bwd(P, dec[hi], g, kNone);
    dskip[hi] = slice(dCat, F[hi], F[hi]);
    TRef dU = slice(dCat, 0, F[hi]);
    const int ci = up[hi];
    // input of the transposed convolution: the activated output of the stage below (or of the bottleneck)
    const TRef Xlow = (lo == L - 1) ? enc[lo].out : dec[lo].out;
    P.macs[CAT_CONV_WGRAD] += (double)N * Ds[lo] * Hs[lo] * Ws[lo] * F[lo] * F[hi] * 8;
    size_wgrad_partials(P, shape_act(P, dU), shape_act(P, Xlow), 2, 2, 1, P.convs[ci].Cop, P.convs[ci].Cip);
    touch(P, P.convs[ci].pw);
    push_op(P.bwd, "wgrad_up2 " + P.convs[ci].name, [&P, ci, Xlow, dU](RunCtx& cx) -> int {
      // dW[ci][co][t] = sum_j X[j][ci] dU[2j + t][co]: the weight gradient of the kernel-2 stride-2 convolution that maps the
      // FINE grid (dU, "input", channels co) to the COARSE grid (X, "output gradient", channels ci): accumulator [T][pad(Co)][pad(Ci)]
      const ConvLayer& c = P.convs[ci];
      WgradOp op;
  memset(&op, 0, sizeof(op));
      op.a = act_of(P, cx, dU);
      op.dy = act_of(P, cx, Xlow);
      op.ksz = 2; op.stride = 2; op.nopad = 1; op.Cip = c.Cop; op.Cop = c.Cip;
      op.dw = reinterpret_cast<float*>(cx.ws + P.bz_off + c.dw);
      return run_wgrad(P, cx, op);
    });
    const Buf lb = P.bufs[Xlow.buf];
    TRef gX = full(P, new_buf(P, N, lb.D, lb.H, lb.W, F[lo]));
    P.macs[CAT_CONV_DGRAD] += (double)N * Ds[lo] * Hs[lo] * Ws[lo] * F[lo] * F[hi] * 8;
    push_op(P.bwd, "dgrad_up2 " + P.convs[ci].name, [&P, ci, dU, gX](RunCtx& cx) -> int {
      // dX[j][ci] = sum_t sum_co dU[2j + t][co] W[ci][co][t]: a kernel-2 stride-2 unpadded convolution of dU with the mode-3 pack
      const ConvLayer& c = P.convs[ci];
      ConvOp op;
      memset(&op, 0, sizeof(op));
      op.nsrc = 1;
      op.src[0] = conv_src(P, cx, c, dU, true);
      op.Cop = c.Cip;
      op.out = act_of(P, cx, gX);
      LAUNCHED(cx, CAT_CONV_DGRAD, launch_igemm_conv(op, cx.st));
      return OK;
    });
    g = gX;
  }
  // g = gradient of the bottleneck output; encoder, bottom to top: skip gradient + gradient through the stride-2 conv below
  TRef gdown = kNone;
  for (int i = L - 1; i >= 0; --i) {
    TRef g1 = (i == L - 1) ? g : dskip[i];
    TRef g2 = (i == L - 1) ? kNone : gdown;
    gdown = build_dyn_block_bwd(P, enc[i], g1, g2);
    // decoder, bottleneck and (six-level nets) the level above it are done
    if (i == (L >= 4 ? L - 2 : L - 1) && i > 0) emit_bwd_split(P);
  }
  emit_unpack_wgrads(P);
  return finish_build(P);
}

static int build(Plan& P) { return P.d.arch == 1 ? build_dynunet(P) : build_unet3d(P); }

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

static int run_backward(b200unet_plan* plan, const float* dlogits, const float* const* params, float* const* grads, void* workspace,
                        void* stream, int part) {
  if (!plan || !dlogits || !params || !grads || !workspace) { set_error("plan_backward: null argument"); return E_INVALID; }
  if (plan->infer) { set_error("plan_backward: this plan was created with inference_only=1 (no backward schedule)"); return E_INVALID; }
  if (part >= 0 && (plan->bwd_split < 0 || part > 1)) {
    set_error("plan_backward_part: part %d of a schedule with %d part(s)", part, plan->bwd_split < 0 ? 1 : 2);
    return E_INVALID;
  }
  RunCtx cx(workspace, stream, plan->prof);
  cx.params = params; cx.grads = grads; cx.dlogits = dlogits;
  cx.part = part;
  if (plan->have_drop) cx.drop = reinterpret_cast<float*>(cx.ws + plan->drop_off);
  const size_t first = part == 1 ? (size_t)plan->bwd_split : 0;
  const size_t last = part == 0 ? (size_t)plan->bwd_split : plan->bwd.size();
  return run_ops(*plan, plan->bwd, first, last, cx, "plan_backward");
}

int b200unet_plan_backward(b200unet_plan* plan, const float* dlogits, const float* const* params, float* const* grads,
                           void* workspace, void* stream) {
  return run_backward(plan, dlogits, params, grads, workspace, stream, -1);
}

int b200unet_plan_input_grad(b200unet_plan* plan, float* dx, void* workspace, void* stream) {
  if (!plan || !dx || !workspace) { set_error("plan_input_grad: null argument"); return E_INVALID; }
  if (!plan->input_grad) { set_error("plan_input_grad: this plan was created without input_grad=1"); return E_INVALID; }
  RunCtx cx(workspace, stream, plan->prof);
  cx.dx = dx;
  return run_ops(*plan, plan->igrad, 0, plan->igrad.size(), cx, "plan_input_grad");
}

int b200unet_plan_backward_parts(const b200unet_plan* plan) { return (!plan || plan->infer) ? 0 : plan->bwd_split >= 0 ? 2 : 1; }

int b200unet_plan_param_backward_part(const b200unet_plan* plan, int i) {
  if (!plan || i < 0 || i >= (int)plan->params.size()) return -1;
  return param_part(*plan, i);
}

int b200unet_plan_backward_part(b200unet_plan* plan, int part, const float* dlogits, const float* const* params, float* const* grads,
                                void* workspace, void* stream) {
  if (part < 0) { set_error("plan_backward_part: part %d", part); return E_INVALID; }
  return run_backward(plan, dlogits, params, grads, workspace, stream, part);
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
