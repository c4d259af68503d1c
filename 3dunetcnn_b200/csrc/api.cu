// extern "C" surface of libb200unet (see include/b200unet.h): argument marshalling only.
#include <cstdarg>
#include <cstring>

#include <cstdlib>
#include "kernels.h"
#include "../../include/b200unet.h"
#include "../../include/b200unet_diag.h"

namespace b200 {
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

// opt-in (common.cuh: launch_pdl)
static const bool kPdlDefault = false;
bool pdl_enabled() {
  static const bool on = getenv("B200UNET_PDL") ? atoi(getenv("B200UNET_PDL")) != 0 : kPdlDefault;
  return on;
}

static Act to_act(const b200unet_tensor* t) {
  return make_act(reinterpret_cast<bf16*>(t->hi), reinterpret_cast<bf16*>(t->lo), t->n, t->d, t->h, t->w, t->c, t->ld);
}
static cudaStream_t to_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// b200unet_conv_desc (+ the diagnostics options) -> ConvOp; the residual and norm-input views live beside the op
struct ConvOpHolder {
  ConvOp op;
  Act res, gx;
};
static int to_conv_op(const b200unet_conv_desc* d, const b200unet_diag_ext* ext, ConvOpHolder* h) {
  ConvOp& op = h->op;
  memset(&op, 0, sizeof(op));
  op.nsrc = d->nsrc;
  if (d->nsrc < 1 || d->nsrc > 2) { set_error("conv3d: nsrc=%d", d->nsrc); return E_INVALID; }
  for (int s = 0; s < d->nsrc; ++s) {
    op.src[s].x = to_act(&d->x[s]);
    op.src[s].w_hi = reinterpret_cast<const bf16*>(d->w_hi[s]);
    op.src[s].w_lo = reinterpret_cast<const bf16*>(d->w_lo[s]);
    op.src[s].ksz = d->ksz[s]; op.src[s].stride = d->stride[s]; op.src[s].Cip = d->cip[s];
    op.src[s].nopad = d->ksz[s] == 2 ? 1 : 0;   // kernel 2 = the unpadded kernel = stride case
  }
  op.Cop = d->cop;
  op.out = to_act(&d->out);
  if (d->res) { h->res = to_act(d->res); op.res = &h->res; }
  op.scale = d->scale; op.stats = d->stats; op.stats_ld = d->stats_ld; op.mode = d->mode;
  if (d->gn_x) { h->gx = to_act(d->gn_x); op.gn_x = &h->gx; }
  op.coef = d->coef; op.coef_ld = d->coef_ld; op.slope = d->slope; op.bstats = d->bstats;
  op.cls_mode = d->cls_mode;
  if (ext) {
    op.bias = ext->bias;
    op.zero_last = ext->zero_last;
    op.max_ctas = ext->max_ctas;
    op.tile128 = ext->tile128;
    for (int s = 0; s < d->nsrc; ++s) {
      op.src[s].x.vD = ext->x_vis[s][0]; op.src[s].x.vH = ext->x_vis[s][1]; op.src[s].x.vW = ext->x_vis[s][2];
    }
  }
  return OK;
}

static void set_vis(Act& a, const int32_t* v) { a.vD = v[0]; a.vH = v[1]; a.vW = v[2]; }

static WgradOp to_wgrad_op(const b200unet_tensor* a, const b200unet_tensor* dy, int ksz, int stride, int cip, int cop,
                           const b200unet_diag_ext* ext) {
  WgradOp op;
  memset(&op, 0, sizeof(op));
  op.a = to_act(a); op.dy = to_act(dy); op.ksz = ksz; op.stride = stride; op.nopad = ksz == 2 ? 1 : 0; op.Cip = cip; op.Cop = cop;
  if (ext) { set_vis(op.a, ext->a_vis); set_vis(op.dy, ext->dy_vis); }
  return op;
}
}  // namespace b200

using namespace b200;

#define NOT_NULL(p)                                                   \
  do {                                                                \
    if (!(p)) { set_error("%s: null argument " #p, __func__); return E_INVALID; } \
  } while (0)

extern "C" {

int b200unet_version(void) { return 106; }
const char* b200unet_last_error(void) { return get_error(); }

int b200unet_ncdhw_to_ndhwc(const float* x, int c_real, const b200unet_tensor* out, void* stream) {
  NOT_NULL(x); NOT_NULL(out);
  return launch_ncdhw_to_act(x, c_real, to_act(out), to_stream(stream));
}
int b200unet_ndhwc_to_ncdhw(const b200unet_tensor* in, int c_real, float* y, void* stream) {
  NOT_NULL(in); NOT_NULL(y);
  return launch_act_to_ncdhw(to_act(in), c_real, y, to_stream(stream));
}
int b200unet_pack_weights(const float* w, int co, int ci, int cop, int cip, int taps, int mode, void* hi, void* lo,
                          void* stream) {
  NOT_NULL(w); NOT_NULL(hi);
  return launch_pack_weights(w, co, ci, cop, cip, taps, mode, reinterpret_cast<bf16*>(hi), reinterpret_cast<bf16*>(lo),
                             to_stream(stream));
}
int b200unet_unpack_wgrad(const float* g, int co, int ci, int cop, int cip, int taps, int mode, float* out,
                          void* stream) {
  NOT_NULL(g); NOT_NULL(out);
  return launch_unpack_wgrad(g, co, ci, cop, cip, taps, mode, out, to_stream(stream));
}

int b200unet_conv3d(const b200unet_conv_desc* d, void* stream) {
  NOT_NULL(d);
  ConvOpHolder h;
  B200_TRY(to_conv_op(d, nullptr, &h));
  return launch_igemm_conv(h.op, to_stream(stream));
}

int b200unet_conv3d_wgrad(const b200unet_tensor* a, const b200unet_tensor* dy, int ksz, int stride, int cip, int cop,
                          float* dw, void* stream) {
  NOT_NULL(a); NOT_NULL(dy); NOT_NULL(dw);
  WgradOp op = to_wgrad_op(a, dy, ksz, stride, cip, cop, nullptr);
  op.dw = dw;
  return launch_wgrad(op, to_stream(stream));
}

int b200unet_gn_apply(const b200unet_tensor* x, const b200unet_tensor* y, const double* stats, const float* gamma,
                      const float* beta, int c, int groups, float eps, float slope, float* coef, void* stream) {
  NOT_NULL(x); NOT_NULL(y); NOT_NULL(stats); NOT_NULL(coef);
  return launch_gn_apply(to_act(x), to_act(y), stats, gamma, beta, c, groups, (long long)x->d * x->h * x->w, eps, coef, slope,
                         to_stream(stream));
}
int b200unet_gn_bwd_finalize(const double* bstats, const float* coef, const float* gamma, int n, int c, int c_ld,
                             int groups, int64_t spatial, float* coef2, float* dgamma, float* dbeta, void* stream) {
  NOT_NULL(bstats); NOT_NULL(coef); NOT_NULL(coef2);
  return launch_gn_bwd_finalize(bstats, coef, gamma, n, c, c_ld, groups, spatial, coef2, dgamma, dbeta,
                                to_stream(stream));
}
int b200unet_gn_bwd(const b200unet_tensor* dz, const b200unet_tensor* x, const float* coef, const double* bstats,
                    const float* gamma, int c, int groups, float* dgamma, float* dbeta, const b200unet_tensor* add1,
                    const b200unet_tensor* add2, const b200unet_tensor* dx, void* stream) {
  return b200unet_diag_gn_bwd(dz, x, coef, bstats, gamma, c, groups, dgamma, dbeta, add1, add2, dx, nullptr, stream);
}
int b200unet_diag_gn_bwd(const b200unet_tensor* dz, const b200unet_tensor* x, const float* coef, const double* bstats, const float* gamma,
                         int c, int groups, float* dgamma, float* dbeta, const b200unet_tensor* add1, const b200unet_tensor* add2,
                         const b200unet_tensor* dx, const float* scale, void* stream) {
  NOT_NULL(dz); NOT_NULL(x); NOT_NULL(coef); NOT_NULL(bstats); NOT_NULL(dx);
  Act a1, a2;
  if (add1) a1 = to_act(add1);
  if (add2) a2 = to_act(add2);
  return launch_gn_bwd(to_act(dz), to_act(x), coef, bstats, gamma, c, groups, (long long)x->d * x->h * x->w, dgamma, dbeta,
                       add1 ? &a1 : nullptr, add2 ? &a2 : nullptr, to_act(dx), scale, to_stream(stream));
}

int b200unet_act_bwd(const b200unet_tensor* g1, const b200unet_tensor* g2, const b200unet_tensor* c, const float* coef, float slope,
                     const b200unet_tensor* dz, double* bstats, int bstats_ld, void* stream) {
  NOT_NULL(g1); NOT_NULL(c); NOT_NULL(coef); NOT_NULL(dz); NOT_NULL(bstats);
  Act a2;
  if (g2) a2 = to_act(g2);
  return launch_act_bwd(to_act(g1), g2 ? &a2 : nullptr, to_act(c), coef, slope, to_act(dz), bstats, bstats_ld, to_stream(stream));
}

int b200unet_prelu_apply(const b200unet_tensor* x, const b200unet_tensor* y, const double* stats, const float* gamma,
                         const float* beta, int c, int groups, float eps, const float* slope, const b200unet_tensor* add, float* coef,
                         void* stream) {
  NOT_NULL(x); NOT_NULL(y); NOT_NULL(stats); NOT_NULL(coef); NOT_NULL(slope);
  Act a;
  if (add) a = to_act(add);
  return launch_gn_apply(to_act(x), to_act(y), stats, gamma, beta, c, groups, (long long)x->d * x->h * x->w, eps, coef, 0.f,
                         to_stream(stream), slope, add ? &a : nullptr);
}
size_t b200unet_prelu_bwd_scratch_bytes(const b200unet_tensor* c) { return c ? act_bwd_slope_scratch_bytes(to_act(c)) : 0; }
int b200unet_prelu_bwd(const b200unet_tensor* g1, const b200unet_tensor* g2, const b200unet_tensor* c, const float* coef,
                       const float* slope, const b200unet_tensor* dz, double* bstats, int bstats_ld, const b200unet_tensor* gsum,
                       float* dslope, float* scratch, void* stream) {
  NOT_NULL(g1); NOT_NULL(c); NOT_NULL(coef); NOT_NULL(slope); NOT_NULL(dz); NOT_NULL(bstats); NOT_NULL(dslope); NOT_NULL(scratch);
  Act a2, gs;
  if (g2) a2 = to_act(g2);
  if (gsum) gs = to_act(gsum);
  return launch_act_bwd(to_act(g1), g2 ? &a2 : nullptr, to_act(c), coef, 0.f, to_act(dz), bstats, bstats_ld, to_stream(stream), slope,
                        dslope, scratch, gsum ? &gs : nullptr);
}
int b200unet_logits_unpack(const b200unet_tensor* in, const b200unet_tensor* add, const float* bias, int c_real, float* logits,
                           void* stream) {
  NOT_NULL(in); NOT_NULL(logits);
  Act a;
  if (add) a = to_act(add);
  return launch_logits_unpack(to_act(in), add ? &a : nullptr, bias, c_real, logits, to_stream(stream));
}

int b200unet_upsample2x_fwd(const b200unet_tensor* x, const b200unet_tensor* y, double* stats, int stats_ld,
                            void* stream) {
  NOT_NULL(x); NOT_NULL(y);
  return launch_upsample2x_fwd(to_act(x), to_act(y), stats, stats_ld, to_stream(stream));
}
int b200unet_upsample2x_add_fwd(const b200unet_tensor* x, const b200unet_tensor* add, const b200unet_tensor* y, double* stats,
                                int stats_ld, void* stream) {
  NOT_NULL(x); NOT_NULL(y);
  Act a;
  if (add) a = to_act(add);
  return launch_upsample2x_fwd(to_act(x), to_act(y), stats, stats_ld, to_stream(stream), add ? &a : nullptr);
}
int b200unet_upsample2x_bwd(const b200unet_tensor* dy, const b200unet_tensor* dx, void* stream) {
  NOT_NULL(dy); NOT_NULL(dx);
  return launch_upsample2x_bwd(to_act(dy), to_act(dx), to_stream(stream));
}
int b200unet_zero_insert(const b200unet_tensor* x, const b200unet_tensor* z, int od, int oh, int ow, void* stream) {
  NOT_NULL(x); NOT_NULL(z);
  return launch_zero_insert(to_act(x), to_act(z), od, oh, ow, to_stream(stream));
}

int b200unet_head_fwd(const b200unet_tensor* x, const float* w, int n_out, int act, float* logits, void* stream) {
  NOT_NULL(x); NOT_NULL(w); NOT_NULL(logits);
  return launch_head_fwd(to_act(x), w, n_out, act, logits, to_stream(stream));
}
size_t b200unet_head_bwd_scratch_bytes(int n_out, int c) { return head_bwd_scratch_bytes(n_out, c); }
int b200unet_head_bwd(const b200unet_tensor* x, const float* w, int n_out, const float* dlogits,
                      const b200unet_tensor* dx, float* dw, float* scratch, void* stream) {
  NOT_NULL(x); NOT_NULL(w); NOT_NULL(dlogits); NOT_NULL(dx); NOT_NULL(dw); NOT_NULL(scratch);
  return launch_head_bwd(to_act(x), w, n_out, dlogits, to_act(dx), dw, to_stream(stream), scratch);
}

static DiceCEDesc to_dice_ce(const b200unet_dice_ce_desc* d) {
  DiceCEDesc r;
  r.act = d->act; r.target_kind = d->target_kind; r.include_background = d->include_background; r.squared_pred = d->squared_pred;
  r.jaccard = d->jaccard; r.batch = d->batch; r.reduction = d->reduction;
  r.smooth_nr = d->smooth_nr; r.smooth_dr = d->smooth_dr; r.lambda_dice = d->lambda_dice; r.lambda_ce = d->lambda_ce;
  r.overlap = d->overlap; r.tversky_alpha = d->tversky_alpha; r.tversky_beta = d->tversky_beta; r.w_type = d->w_type;
  r.voxel_term = d->voxel_term; r.focal_softmax = d->focal_softmax; r.focal_gamma = d->focal_gamma; r.focal_alpha = d->focal_alpha;
  r.focal_use_alpha = d->focal_use_alpha; r.class_weight = d->class_weight; r.hdt_weight = d->hdt_weight;
  return r;
}
int b200unet_dice_fwd(const b200unet_dice_ce_desc* desc, const float* logits, const void* target, int n, int c, int64_t spatial,
                      double* scratch, float* loss, void* stream) {
  NOT_NULL(desc); NOT_NULL(logits); NOT_NULL(target); NOT_NULL(scratch); NOT_NULL(loss);
  return launch_dice_fwd(to_dice_ce(desc), logits, target, n, c, spatial, scratch, loss, to_stream(stream));
}
int b200unet_dice_bwd(const b200unet_dice_ce_desc* desc, const float* logits, const void* target, int n, int c, int64_t spatial,
                      const double* scratch, const float* grad_out, float* dlogits, void* stream) {
  NOT_NULL(desc); NOT_NULL(logits); NOT_NULL(target); NOT_NULL(scratch); NOT_NULL(grad_out); NOT_NULL(dlogits);
  return launch_dice_bwd(to_dice_ce(desc), logits, target, n, c, spatial, scratch, grad_out, dlogits, to_stream(stream));
}
size_t b200unet_dice_ce_scratch_bytes(const b200unet_dice_ce_desc* desc, int n, int c, int64_t spatial) {
  if (!desc) { set_error("%s: null argument desc", __func__); return 0; }
  return dice_ce_scratch_bytes(to_dice_ce(desc), n, c, spatial);
}
int b200unet_dice_ce_fwd(const b200unet_dice_ce_desc* desc, const float* logits, const void* target, int n, int c, int64_t spatial,
                         void* scratch, float* loss, void* stream) {
  NOT_NULL(desc); NOT_NULL(logits); NOT_NULL(target); NOT_NULL(scratch); NOT_NULL(loss);
  return launch_dice_ce_fwd(to_dice_ce(desc), logits, target, n, c, spatial, scratch, loss, to_stream(stream));
}
int b200unet_dice_ce_bwd(const b200unet_dice_ce_desc* desc, const float* logits, const void* target, int n, int c, int64_t spatial,
                         const void* scratch, const float* grad_out, float* dlogits, void* stream) {
  NOT_NULL(desc); NOT_NULL(logits); NOT_NULL(target); NOT_NULL(scratch); NOT_NULL(grad_out); NOT_NULL(dlogits);
  return launch_dice_ce_bwd(to_dice_ce(desc), logits, target, n, c, spatial, scratch, grad_out, dlogits, to_stream(stream));
}

size_t b200unet_hausdorff_dt_scratch_bytes(const b200unet_dice_ce_desc* desc, int n, int c, int d, int h, int w) {
  if (!desc) { set_error("%s: null argument desc", __func__); return 0; }
  return hausdorff_dt_scratch_bytes(to_dice_ce(desc), n, c, d, h, w);
}
int b200unet_hausdorff_dt_weight(const b200unet_dice_ce_desc* desc, const float* logits, const void* target, int n, int c, int d, int h,
                                 int w, float alpha, void* scratch, float* weight, void* stream) {
  NOT_NULL(desc); NOT_NULL(logits); NOT_NULL(target); NOT_NULL(scratch); NOT_NULL(weight);
  return launch_hausdorff_dt_fields(to_dice_ce(desc), logits, target, n, c, d, h, w, alpha, scratch, weight, nullptr, nullptr,
                                    to_stream(stream));
}
int b200unet_diag_hausdorff_dt_fields(const b200unet_dice_ce_desc* desc, const float* logits, const void* target, int n, int c, int d,
                                      int h, int w, void* scratch, float* pred_field, float* target_field, void* stream) {
  NOT_NULL(desc); NOT_NULL(logits); NOT_NULL(target); NOT_NULL(scratch);
  return launch_hausdorff_dt_fields(to_dice_ce(desc), logits, target, n, c, d, h, w, 1.f, scratch, nullptr, pred_field, target_field,
                                    to_stream(stream));
}

int b200unet_tiles_gather(const float* vol, int n, int c, int d, int h, int w, const int32_t* starts, int ntiles, int rd, int rh,
                          int rw, float* tiles, void* stream) {
  NOT_NULL(vol); NOT_NULL(starts); NOT_NULL(tiles);
  return launch_tiles_gather(vol, n, c, d, h, w, starts, ntiles, rd, rh, rw, tiles, to_stream(stream));
}
int b200unet_tiles_scatter(const float* pred, int c, const int32_t* starts, int ntiles, int rd, int rh, int rw,
                           const float* importance, float* out, int n, int d, int h, int w, void* stream) {
  NOT_NULL(pred); NOT_NULL(starts); NOT_NULL(importance); NOT_NULL(out);
  return launch_tiles_scatter(pred, c, starts, ntiles, rd, rh, rw, importance, out, n, d, h, w, to_stream(stream));
}
int b200unet_tiles_count(const int32_t* starts_d, int nd, const int32_t* starts_h, int nh, const int32_t* starts_w, int nw, int rd,
                         int rh, int rw, const float* importance, float* cnt, int d, int h, int w, void* stream) {
  return launch_tiles_count(starts_d, nd, starts_h, nh, starts_w, nw, rd, rh, rw, importance, cnt, d, h, w, to_stream(stream));
}
int b200unet_tiles_normalize(float* out, const float* cnt, int nc, int64_t spatial, void* stream) {
  NOT_NULL(out); NOT_NULL(cnt);
  return launch_tiles_normalize(out, cnt, nc, spatial, to_stream(stream));
}
int b200unet_one_hot(const float* data, int n, int64_t spatial, const float* values, const int32_t* begin, int n_channels,
                     int do_round, uint8_t* y, void* stream) {
  return launch_one_hot(data, n, spatial, values, begin, n_channels, do_round, y, to_stream(stream));
}
int b200unet_zscore(const float* x, int groups, int64_t spatial, int nonzero, double* stats, float* y, void* stream) {
  return launch_zscore(x, groups, spatial, nonzero, stats, y, to_stream(stream));
}
int b200unet_label_map(const float* p, int n_labels, int64_t spatial, const int32_t* labels, int act, float threshold,
                       int hierarchy, int sum_then_threshold, int16_t* out, void* stream) {
  return launch_label_map(p, n_labels, spatial, labels, act, threshold, hierarchy, sum_then_threshold, out, to_stream(stream));
}

size_t b200unet_augment_scratch_bytes(int n, int c, int64_t spatial) { return augment_scratch_bytes(n, c, spatial); }
int b200unet_augment_resample(const float* image, const uint8_t* label, int n, int c, int l, int d, int h, int w, const float* affine,
                              int padding, int nonzero, float* image_out, uint8_t* label_out, void* scratch, void* stream) {
  return launch_augment_resample(image, label, n, c, l, d, h, w, affine, padding, nonzero, image_out, label_out, scratch,
                                 to_stream(stream));
}
int b200unet_augment_intensity(float* image, int n, int c, int64_t spatial, int normalize, int nonzero, int channel_wise,
                               const float* coef, void* scratch, void* stream) {
  return launch_augment_intensity(image, n, c, spatial, normalize, nonzero, channel_wise, coef, scratch, to_stream(stream));
}
static_assert(sizeof(AugSample) == 5 * sizeof(int64_t), "b200unet.h sample rows are five int64");
size_t b200unet_foreground_scratch_bytes(int n, int c) { return foreground_scratch_bytes(n, c); }
int b200unet_foreground_box(const int64_t* samples, int n, int c, int64_t max_spatial, int crop, const int64_t* ranks,
                            const float* gamma, int margin, int allow_smaller, const double* affine, int d, int h, int w,
                            float* affine_out, int32_t* box, int32_t* empty, float* threshold, void* scratch, void* stream) {
  return launch_foreground_box(reinterpret_cast<const AugSample*>(samples), n, c, max_spatial, crop,
                               reinterpret_cast<const long long*>(ranks), gamma, margin, allow_smaller, affine, d, h, w, affine_out,
                               box, empty, threshold, scratch, to_stream(stream));
}
int b200unet_augment_resample_samples(const int64_t* samples, int n, int c, int l, int d, int h, int w, const float* affine,
                                      int padding, int nonzero, float* image_out, uint8_t* label_out, void* scratch, void* stream) {
  return launch_augment_resample_samples(reinterpret_cast<const AugSample*>(samples), n, c, l, d, h, w, affine, padding, nonzero,
                                         image_out, label_out, scratch, to_stream(stream));
}

int b200unet_resample_to_grid(const float* src, int c, int sd, int sh, int sw, const double affine[12], int mode, float* dst, int dd,
                              int dh, int dw, void* stream) {
  NOT_NULL(src); NOT_NULL(affine); NOT_NULL(dst);
  IndexAffine m;
  memcpy(m.m, affine, sizeof(m.m));
  return launch_resample_to_grid(src, c, sd, sh, sw, m, mode, dst, dd, dh, dw, to_stream(stream));
}

size_t b200unet_cc_scratch_bytes(int nvol, int d, int h, int w) { return cc_scratch_bytes(nvol, d, h, w); }
int b200unet_cc_label(const uint8_t* mask, int nvol, int d, int h, int w, int connectivity, int32_t* labels, int32_t* counts,
                      void* scratch, void* stream) {
  NOT_NULL(mask); NOT_NULL(labels); NOT_NULL(counts); NOT_NULL(scratch);
  return launch_cc_label(mask, nvol, d, h, w, connectivity, labels, counts, scratch, to_stream(stream));
}
int b200unet_cc_sort_by_size(int32_t* labels, int nvol, int d, int h, int w, int max_count, void* scratch, void* stream) {
  NOT_NULL(labels); NOT_NULL(scratch);
  return launch_cc_sort_by_size(labels, nvol, d, h, w, max_count, scratch, to_stream(stream));
}

static SurfaceMask to_surface_mask(const b200unet_surface_mask* m) {
  SurfaceMask s;
  s.data = m->data;
  s.dtype = m->dtype;
  for (int i = 0; i < 5; ++i) s.stride[i] = m->stride[i];
  return s;
}
size_t b200unet_surface_scratch_bytes(int b, int c, int d, int h, int w) { return surface_scratch_bytes(b, c, d, h, w); }
int b200unet_surface_distance(const b200unet_surface_mask* pred, const b200unet_surface_mask* gt, int b, int c, int d, int h, int w,
                              const double* spacing, float q, int hd_dirs, int asd_dirs, const float* tau, float* hd, float* asd,
                              float* nsd, void* scratch, void* stream) {
  NOT_NULL(pred); NOT_NULL(gt); NOT_NULL(spacing); NOT_NULL(scratch);
  return launch_surface_distance(to_surface_mask(pred), to_surface_mask(gt), b, c, d, h, w, spacing, q, hd_dirs, asd_dirs, tau, hd, asd,
                                 nsd, scratch, to_stream(stream));
}

static OverlapOperand to_overlap_operand(const b200unet_overlap_operand* o) {
  OverlapOperand r;
  r.data = o->data;
  r.kind = o->kind;
  r.dtype = o->dtype;
  r.thr = o->threshold;
  return r;
}
int b200unet_overlap_counts(const b200unet_overlap_operand* pred, const b200unet_overlap_operand* gt, int b, int c, int d, int h,
                            int w, int64_t* counts, void* stream) {
  NOT_NULL(pred); NOT_NULL(gt); NOT_NULL(counts);
  return launch_overlap_counts(to_overlap_operand(pred), to_overlap_operand(gt), b, c, d, h, w, counts, to_stream(stream));
}

// ---- diagnostics (include/b200unet_diag.h)
int b200unet_diag_conv3d_route(const b200unet_conv_desc* desc, const b200unet_diag_ext* ext, b200unet_conv_route* route) {
  NOT_NULL(desc); NOT_NULL(route);
  ConvOpHolder h;
  B200_TRY(to_conv_op(desc, ext, &h));
  ConvRoute r;
  B200_TRY(conv_route(h.op, device_sms(), &r));
  route->kind = r.kind; route->bn = r.BN; route->kc = r.KC;
  route->kchunks[0] = r.kchunks[0]; route->kchunks[1] = r.kchunks[1];
  route->npass = r.npass; route->cls_pair = r.cls_pair;
  route->tw = r.tw; route->th = r.th; route->td = r.td;
  for (int i = 0; i < 3; ++i) route->grid[i] = r.grid[i];
  route->stages = r.stages; route->blocks_per_sm = r.blocks_per_sm; route->smem_bytes = r.smem_bytes;
  route->wgs = r.wgs;
  return OK;
}

int b200unet_diag_wgrad_route(const b200unet_tensor* a, const b200unet_tensor* dy, int ksz, int stride, int cip, int cop,
                              const b200unet_diag_ext* ext, int deterministic, int num_sms, b200unet_wgrad_route* route) {
  NOT_NULL(a); NOT_NULL(dy); NOT_NULL(route);
  if (num_sms < 1) { set_error("%s: num_sms=%d", __func__, num_sms); return E_INVALID; }
  WgradOp op = to_wgrad_op(a, dy, ksz, stride, cip, cop, ext);
  float placeholder;
  if (deterministic) op.part = &placeholder;   // only its presence matters to the route
  WgradRoute r;
  B200_TRY(wgrad_route(op, num_sms, &r));
  route->kind = r.kind; route->ci8 = r.ci8;
  route->cb = r.CB; route->bn = r.BN; route->qt = r.QT;
  route->groups = r.groups; route->cotiles = r.cotiles; route->kblocks = r.kblocks; route->splits = r.splits; route->npass = r.npass;
  route->tw = r.tw; route->th = r.th; route->td = r.td;
  route->part_bytes = (int64_t)r.part_bytes;
  route->ctas = r.ctas;
  return OK;
}

size_t b200unet_diag_wgrad_partial_bytes(const b200unet_tensor* a, const b200unet_tensor* dy, int ksz, int stride, int cip, int cop,
                                         const b200unet_diag_ext* ext, int num_sms) {
  if (!a || !dy || num_sms < 1) { set_error("%s: bad argument", __func__); return 0; }
  return wgrad_partial_bytes(to_wgrad_op(a, dy, ksz, stride, cip, cop, ext), num_sms);
}

int b200unet_diag_conv3d_ex(const b200unet_conv_desc* desc, const b200unet_diag_ext* ext, void* stream) {
  NOT_NULL(desc);
  ConvOpHolder h;
  B200_TRY(to_conv_op(desc, ext, &h));
  return launch_igemm_conv(h.op, to_stream(stream));
}

// the weight gradient as the plans run it (plan.cu: run_wgrad)
int b200unet_diag_wgrad_ex(const b200unet_tensor* a, const b200unet_tensor* dy, int ksz, int stride, int cip, int cop,
                           const b200unet_diag_ext* ext, float* part, size_t part_bytes, int* splits, float* dw, void* stream) {
  NOT_NULL(a); NOT_NULL(dy); NOT_NULL(dw);
  WgradOp op = to_wgrad_op(a, dy, ksz, stride, cip, cop, ext);
  op.dw = dw;
  if (!part) return launch_wgrad(op, to_stream(stream));
  int n = 0;
  op.part = part; op.part_bytes = part_bytes; op.part_splits = &n;
  B200_TRY(launch_wgrad(op, to_stream(stream)));
  B200_REQUIRE(n >= 1, E_INVALID, "wgrad: deterministic weight gradient wrote no partial slots");
  if (splits) *splits = n;
  return launch_wgrad_reduce(part, n, (long long)ksz * ksz * ksz * cip * cop, dw, to_stream(stream));
}

int b200unet_diag_bias_grad(const b200unet_tensor* dy, const b200unet_diag_ext* ext, float* scratch, float* dbias, void* stream) {
  NOT_NULL(dy); NOT_NULL(scratch); NOT_NULL(dbias);
  Act y = to_act(dy);
  if (ext) set_vis(y, ext->dy_vis);
  return launch_bias_grad(y, dbias, scratch, to_stream(stream));
}
size_t b200unet_diag_bias_grad_scratch_bytes(int c) { return bias_grad_scratch_bytes(c); }

int b200unet_diag_head_fwd(const b200unet_tensor* x, const float* w, const float* bias, int n_out, int act, float* logits, void* stream) {
  NOT_NULL(x); NOT_NULL(w); NOT_NULL(logits);
  return launch_head_fwd(to_act(x), w, n_out, act, logits, to_stream(stream), bias);
}
int b200unet_diag_head_bwd(const b200unet_tensor* x, const float* w, int n_out, const float* dlogits, const b200unet_tensor* dx, float* dw,
                           float* dbias, float* scratch, void* stream) {
  NOT_NULL(x); NOT_NULL(w); NOT_NULL(dlogits); NOT_NULL(dx); NOT_NULL(dw); NOT_NULL(scratch);
  return launch_head_bwd(to_act(x), w, n_out, dlogits, to_act(dx), dw, to_stream(stream), scratch, dbias);
}
int b200unet_diag_head_dbias(const float* dlogits, int n, int n_out, int64_t spatial, float* scratch, float* dbias, void* stream) {
  NOT_NULL(dlogits); NOT_NULL(scratch); NOT_NULL(dbias);
  return launch_head_dbias(dlogits, n, n_out, spatial, dbias, to_stream(stream), scratch);
}
int b200unet_diag_input_pack(const float* x, int c, const b200unet_tensor* out, double* stats, int stats_ld, void* stream) {
  NOT_NULL(x); NOT_NULL(out);
  return launch_input_pack(x, c, to_act(out), stats, stats_ld, to_stream(stream));
}
int b200unet_diag_input_grad(const b200unet_tensor* dz, const b200unet_tensor* x, const float* coef, const float* coef2, int coef_ld,
                             const b200unet_tensor* r, int c, float* dx, void* stream) {
  NOT_NULL(r); NOT_NULL(dx);
  Act a, b;
  if (dz) {
    NOT_NULL(x);
    a = to_act(dz); b = to_act(x);
  }
  return launch_input_grad(dz ? &a : nullptr, dz ? &b : nullptr, coef, coef2, coef_ld, to_act(r), c, dx, to_stream(stream));
}

}  // extern "C"
