// Internal kernel launchers of libb200unet (host API; all asynchronous on the given stream).
#pragma once
#include "common.cuh"

namespace b200 {

// ---- bandwidth-bound kernels (elementwise.cu)
int launch_input_pack(const float* x, int C, const Act& out, double* stats, int stats_ld, cudaStream_t st);
// GroupNorm(+ReLU / LeakyReLU) forward: statistics -> coefficients (coef [N][x.C][4], written) -> y; x.C <= 1024
// slope_dev (optional): the negative slope is read from this device scalar (a learnable PReLU) instead of `slope`;
// add (optional, y's shape): y = act(A x + B) + add, the addend read as hi + lo
int launch_gn_apply(const Act& x, const Act& y, const double* stats, const float* gamma, const float* beta, int C, int G,
                    long long S, float eps, float* coef, float slope, cudaStream_t st, const float* slope_dev = nullptr,
                    const Act* add = nullptr);
// GroupNorm backward: backward statistics -> (E, F), dgamma, dbeta -> dx; x.C <= 1024
int launch_gn_bwd(const Act& dz, const Act& x, const float* coef, const double* bstats, const float* gamma, int C, int G,
                  long long S, float* dgamma, float* dbeta, const Act* add1, const Act* add2, const Act& dx,
                  const float* scale, cudaStream_t st);
// the same without dx (the first block's norm): dgamma, dbeta and (E, F) into coef2 [N][Cld][2] for launch_input_grad
int launch_gn_bwd_finalize(const double* bstats, const float* coef, const float* gamma, int N, int C, int Cld, int G,
                           long long S, float* coef2, float* dgamma, float* dbeta, cudaStream_t st);
int launch_upsample2x_fwd(const Act& x, const Act& y, double* stats, int stats_ld, cudaStream_t st, const Act* add = nullptr);
int launch_upsample2x_bwd(const Act& dy, const Act& dx, cudaStream_t st);
// The 1x1x1 head takes 1..B200_HEAD_MAX_OUTPUTS outputs: 1..8 run the SIMT kernels below with fp32 weights, 9..128 the
// tensor-core kernels of head.cu (launch_head_mma_*), chosen inside launch_head_fwd / launch_head_bwd from n_out alone.
#define B200_HEAD_MAX_OUTPUTS 128
int launch_head_fwd(const Act& x, const float* w, int n_out, int act_mode, float* logits, cudaStream_t st,
                    const float* bias = nullptr);
int launch_head_dbias(const float* dlogits, int N, int NO, long long S, float* dbias, cudaStream_t st, float* scratch);
// post-activation blocks: dz = (g1 [+ g2]) * act'(A c + B), bstats += (sum dz, sum dz*xhat)
// PReLU (optional): slope_dev as in launch_gn_apply; dslope (with scratch of act_bwd_slope_scratch_bytes(c)) = sum over z <= 0
// of z * (g1 [+ g2]), written, bit-identical run to run (per-block partials + a fixed-order sum); gsum = g1 [+ g2]
int launch_act_bwd(const Act& g1, const Act* g2, const Act& c, const float* coef, float slope, const Act& dz, double* bstats,
                   int bstats_ld, cudaStream_t st, const float* slope_dev = nullptr, float* dslope = nullptr,
                   float* scratch = nullptr, const Act* gsum = nullptr);
size_t act_bwd_slope_scratch_bytes(const Act& c);
// fp32 NCDHW logits [N][C][S] = in (+ bias[c]) (+ add) over the C real channels of the padded conv result `in`
int launch_logits_unpack(const Act& in, const Act* add, const float* bias, int C, float* y, cudaStream_t st);
// scratch: head_bwd_scratch_bytes(n_out, C) (per-block partial sums).  dbias (more than 8 outputs only; launch_head_dbias
// serves 1..8): also write the bias gradient from the same pass.
int launch_head_bwd(const Act& x, const float* w, int n_out, const float* dlogits, const Act& dx, float* dw,
                    cudaStream_t st, float* scratch, float* dbias = nullptr);
size_t head_bwd_scratch_bytes(int n_out, int C);
// ---- tensor-core head, 9..128 outputs, C a multiple of 8 up to 64 (head.cu)
int launch_head_mma_fwd(const Act& x, const float* w, int n_out, int act_mode, float* logits, cudaStream_t st, const float* bias);
// writes the per-CTA partial sums (weight gradient, then bias gradient when want_dbias) of *slots CTAs into part
int launch_head_mma_bwd(const Act& x, const float* w, int n_out, const float* dlogits, const Act& dx, int want_dbias, float* part,
                        int* slots, cudaStream_t st);
size_t head_mma_bwd_scratch_bytes(int n_out, int C);
// ---- weight packing / gradient unpacking (small_ops.cu): shared-memory tiled transposes
// one tensor; Cop and Cip (the padded extents) must be multiples of 8, T <= 27
int launch_pack_weights(const float* w, int Co, int Ci, int Cop, int Cip, int T, int mode, bf16* hi, bf16* lo,
                        cudaStream_t st);
int launch_unpack_wgrad(const float* g, int Co, int Ci, int Cop, int Cip, int T, int mode, float* out,
                        cudaStream_t st);
// batched weight packing / gradient unpacking (one launch for the whole network)
struct PtrTable { const void* p[256]; };
// PackJob::mode, the `mode` of b200unet_pack_weights / b200unet_unpack_wgrad.  Conv3d weight [Co][Ci][T]:
enum PackMode {
  PACK_FWD = 0,          // forward [T][Cop][Cip]; unpack: [T][Cip][Cop] accumulator -> [Co][Ci][T]
  PACK_DGRAD = 1,        // data-gradient [T][Cip][Cop], taps flipped
  // ConvTranspose3d weight [Ci][Co][T] (the modes from PACK_T_FLIPPED on):
  PACK_T_FLIPPED = 2,    // forward [T][Cop][Cip], taps flipped (the zero-inserted k3 s2 p1 layer); unpack: -> [Ci][Co][T] flipped
  PACK_T_DGRAD = 3,      // data-gradient [T][Cip][Cop], unflipped
  PACK_T_FWD = 4,        // forward [T][Cop][Cip], unflipped (kernel = stride ConvTranspose3d: out[2j+p] = x[j] w[p])
};
struct PackJob {
  int pidx;                 // index into the parameter / gradient pointer table
  int Co, Ci, Cop, Cip, T;
  int mode;                 // PackMode; unpack: PACK_FWD or PACK_T_FLIPPED
  long long off_hi, off_lo; // workspace byte offsets (unpack: off_hi = fp32 accumulator)
};
int launch_pack_all(const PtrTable& params, const PackJob* jobs_dev, int njobs, uint8_t* ws, bool split, cudaStream_t st);
int launch_unpack_all(const PtrTable& grads, const PackJob* jobs_dev, int njobs, const uint8_t* ws, cudaStream_t st);
// dbias[c] = sum over the VISIBLE voxels of dy (overwritten), in a fixed order, for the first c_real channels (<= 0: all
// dy.C); scratch: bias_grad_scratch_bytes(dy.C)
int launch_bias_grad(const Act& dy, float* dbias, float* scratch, cudaStream_t st, int c_real = 0);
size_t bias_grad_scratch_bytes(int C);
int launch_zero_insert(const Act& x, const Act& z, int od, int oh, int ow, cudaStream_t st);
int launch_ncdhw_to_act(const float* x, int C, const Act& out, cudaStream_t st);
int launch_act_to_ncdhw(const Act& in, int C, float* y, cudaStream_t st);
// gradient of the network input, NCDHW fp32 [N][C][S]: dx = (A dz + E x + F) + r over the C real channels (coef [N][coef_ld][4],
// coef2 [N][coef_ld][2] as left by the GroupNorm backward); dz == nullptr: dx = r (the layout transpose alone)
int launch_input_grad(const Act* dz, const Act* x, const float* coef, const float* coef2, int coef_ld, const Act& r, int C, float* dx,
                      cudaStream_t st);

// ---- Dice criteria: the options of both; the fields mirror b200unet_dice_ce_desc
enum TargetKind { T_LABEL_U8 = 0, T_LABEL_I64 = 1, T_ONEHOT_U8 = 2, T_SOFT_F32 = 3 };
enum ActKind { A_NONE = 0, A_SIGMOID = 1, A_SOFTMAX = 2 };
enum OverlapKind { O_DICE = 0, O_TVERSKY = 1, O_GDICE = 2 };
enum GDiceWeight { W_SQUARE = 0, W_SIMPLE = 1, W_UNIFORM = 2 };
enum VoxelTerm { V_CE = 0, V_FOCAL = 1 };
struct DiceCEDesc {
  int act;               // ActKind: 0 identity, 1 sigmoid, 2 softmax over channels
  int target_kind;       // TargetKind: 0 uint8 label map [N][1][S], 1 int64 label map, 2 uint8 [N][C][S], 3 fp32 [N][C][S]
  int include_background, squared_pred, jaccard, batch;
  int reduction;         // 0 mean, 1 sum
  float smooth_nr, smooth_dr, lambda_dice, lambda_ce;
  // a zeroed tail is the Dice overlap with the CE term
  int overlap;           // OverlapKind
  float tversky_alpha, tversky_beta;
  int w_type;            // GDiceWeight
  int voxel_term;        // VoxelTerm, scaled by lambda_ce
  int focal_softmax;     // focal: 0 sigmoid form, 1 softmax form over the kept channels
  float focal_gamma, focal_alpha;
  int focal_use_alpha;
  const float* class_weight;   // focal: DEVICE fp32 [C'] (C' = channels kept), nullptr = none
};
// the checks both criteria make: a non-empty shape and in-range options ("who" prefixes the error message)
int check_dice_desc(const DiceCEDesc& d, int N, int C, long long S, const char* who);
// The per-voxel term's total is divided by this: CE: N*S (mean) or 1 (sum); focal: N*C'*S (mean) or S (sum, MONAI's
// FocalLoss averages over the voxels before it sums over samples and classes)
__host__ __device__ inline double voxel_divisor(const DiceCEDesc& d, int N, int C, long long S) {
  if (d.voxel_term == V_CE) return d.reduction == 0 ? (double)N * S : 1.0;
  const int kept = (!d.include_background && C > 1) ? C - 1 : C;
  return d.reduction == 0 ? (double)N * kept * S : (double)S;
}
// The loss and coef [N][C][2] (the backward's dF/dI, dF/dP per (n, c)) from sums [N][C][3] (I, P, T) in one single-block
// launch; ce [N] (the summed per-voxel terms of each sample) is read only when lambda_ce != 0 (dice.cu)
int launch_dice_finalize(const DiceCEDesc& d, const double* sums, const double* ce, int N, int C, long long S, double* coef,
                         float* loss, cudaStream_t st);

// ---- DiceLoss (dice.cu): sigmoid or identity, uint8 or fp32 [N][C][S] target, lambda_ce == 0.  scratch: sums [N][C][3]
// then coef [N][C][2], fp64
int launch_dice_fwd(const DiceCEDesc& d, const float* logits, const void* target, int N, int C, long long S, double* scratch,
                    float* loss, cudaStream_t st);
int launch_dice_bwd(const DiceCEDesc& d, const float* logits, const void* target, int N, int C, long long S, const double* scratch,
                    const float* grad_out, float* dlogits, cudaStream_t st);

// ---- Dice + cross-entropy criterion (dice_ce.cu)
size_t dice_ce_scratch_bytes(const DiceCEDesc& d, int N, int C, long long S);   // 0: the shape or options are rejected
int launch_dice_ce_fwd(const DiceCEDesc& d, const float* logits, const void* target, int N, int C, long long S, void* scratch,
                       float* loss, cudaStream_t st);
int launch_dice_ce_bwd(const DiceCEDesc& d, const float* logits, const void* target, int N, int C, long long S, const void* scratch,
                       const float* grad_out, float* dlogits, cudaStream_t st);

// ---- steps before / after the path (prepost.cu): sliding-window tiles, one-hot targets, z-score, label maps
#define B200_MAX_TILES 16
#define B200_MAX_LABEL_CHANNELS 128
#define B200_MAX_LABEL_VALUES 256   // LabelTable (prepost.cu) stays a ~1.5 KB kernel parameter
int launch_tiles_gather(const float* vol, int N, int C, int D, int H, int W, const int32_t* starts, int ntiles, int rd, int rh,
                        int rw, float* tiles, cudaStream_t st);
int launch_tiles_scatter(const float* pred, int C, const int32_t* starts, int ntiles, int rd, int rh, int rw, const float* imp,
                         float* out, int N, int D, int H, int W, cudaStream_t st);
int launch_tiles_count(const int32_t* sd_dev, int nd, const int32_t* sh_dev, int nh, const int32_t* sw_dev, int nw, int rd, int rh,
                       int rw, const float* imp, float* cnt, int D, int H, int W, cudaStream_t st);
int launch_tiles_normalize(float* out, const float* cnt, int NC, long long S, cudaStream_t st);
int launch_one_hot(const float* data, int N, long long S, const float* values, const int32_t* begin, int n_channels, int do_round,
                   uint8_t* y, cudaStream_t st);
int launch_zscore(const float* x, int groups, long long S, int nonzero, double* stats, float* y, cudaStream_t st);
int launch_label_map(const float* p, int L, long long S, const int32_t* labels, int act, float thr, int hierarchy,
                     int sum_then_threshold, int16_t* out, cudaStream_t st);

// ---- random flips / rotation + z-score + scale / shift of a training batch (augment.cu)
#define B200_AUG_MAX_CHANNELS 16
// scratch: stats [N][C][3] fp64 (sum, sumsq, count), then the per-block partials of the resample pass; 0: the shape is rejected
size_t augment_scratch_bytes(int N, int C, long long S);
// affine: DEVICE [N][12] fp32 row-major 3x4 (output index (d, h, w) -> source index); padding 0 border, 1 zeros; L = 0: no label
int launch_augment_resample(const float* img, const uint8_t* lab, int N, int C, int L, int D, int H, int W, const float* affine,
                            int padding, int nonzero, float* img_out, uint8_t* lab_out, void* scratch, cudaStream_t st);
// one sample of a batch of different extents (DEVICE table, the layout of b200unet.h's sample rows): image [C][d][h][w] fp32,
// label [L][d][h][w] uint8 (nullptr without a label)
struct AugSample {
  const float* img;
  const uint8_t* lab;
  long long d, h, w;
};
// as launch_augment_resample onto the (D, H, W) grid, sample n read from samples[n]
int launch_augment_resample_samples(const AugSample* samples, int N, int C, int L, int D, int H, int W, const float* affine,
                                    int padding, int nonzero, float* img_out, uint8_t* lab_out, void* scratch, cudaStream_t st);
// in place on the resampled image; coef: DEVICE [N][C][2] (a, b)
int launch_augment_intensity(float* img, int N, int C, long long S, int normalize, int nonzero, int channel_wise, const float* coef,
                             void* scratch, cudaStream_t st);

// ---- foreground box of each sample + the composed crop / resize / augmentation affine (foreground.cu)
// scratch: select histograms and state per (sample, channel), box accumulators per sample; 0: the shape is rejected
size_t foreground_scratch_bytes(int N, int C);
// crop = 0: the whole volume; ranks == nullptr: select x > 0; else x > thr with thr per (n, c) the linear interpolation
// (weight gamma[n][c]) of the order statistics ranks[n][c][0..1], written to thr.  affine_in DEVICE fp64 [N][12] on the
// (OD, OH, OW) grid -> affine_out fp32 [N][12] onto the sample's own grid; box int32 [N][3][2] (start, end), empty int32 [N]
int launch_foreground_box(const AugSample* samples, int N, int C, long long max_spatial, int crop, const long long* ranks,
                          const float* gamma, int margin, int allow_smaller, const double* affine_in, int OD, int OH, int OW,
                          float* affine_out, int32_t* box, int32_t* empty, float* thr, void* scratch, cudaStream_t st);

// ---- resample a prediction onto the grid of its image file (resample.cu)
// row-major 3x4 map of target index (d, h, w, 1) -> source index, passed by value
struct IndexAffine { double m[12]; };
// src fp32 [C][sd][sh][sw] -> dst fp32 [C][dd][dh][dw], 1 <= C <= B200_MAX_LABEL_CHANNELS; mode 0 trilinear, 1 nearest; border padding
int launch_resample_to_grid(const float* src, int C, int sd, int sh, int sw, const IndexAffine& m, int mode, float* dst, int dd,
                            int dh, int dw, cudaStream_t st);

// ---- connected components of binary masks (ccl.cu)
size_t cc_scratch_bytes(int nvol, int d, int h, int w);   // 0: the shape is rejected
int launch_cc_label(const uint8_t* mask, int nvol, int d, int h, int w, int connectivity, int32_t* labels, int32_t* counts,
                    void* scratch, cudaStream_t st);
int launch_cc_sort_by_size(int32_t* labels, int nvol, int d, int h, int w, int max_count, void* scratch, cudaStream_t st);

// ---- boundary-distance scores of binary segmentations (surface.cu)
#define B200_SURFACE_MAX_EXTENT 256   // per axis: site indices of the distance transform are uint8, offsets int16
#define B200_SURFACE_MAX_PAIRS 4096   // (item, class) pairs per call
// element (b, c, d, h, w) at data + b stride[0] + c stride[1] + d stride[2] + h stride[3] + w stride[4] (elements); foreground is
// value == 1; dtype 0 = bool / uint8, 1 = fp32.  Field order of b200unet_surface_mask.
struct SurfaceMask {
  const void* data;
  int dtype;
  long long stride[5];
};
size_t surface_scratch_bytes(int nb, int nc, int d, int h, int w);   // 0: the shape is rejected
// spacing DEVICE fp64 [nb][3]; q = 0: Hausdorff is the max, else the fp32 quantile q in (0, 1]; hd_dirs / asd_dirs 1 = pred -> gt,
// 2 = both; tau DEVICE fp32 [nc] (surface Dice thresholds); hd, asd, nsd DEVICE fp32 [nb][nc] or nullptr
int launch_surface_distance(const SurfaceMask& pred, const SurfaceMask& gt, int nb, int nc, int d, int h, int w, const double* spacing,
                            float q, int hd_dirs, int asd_dirs, const float* tau, float* hd, float* asd, float* nsd, void* scratch,
                            cudaStream_t st);

// ---- overlap counts of segmentations: P, G, I per (item, class) (overlap.cu)
#define B200_OVERLAP_MAX_CLASSES 128
#define B200_OVERLAP_MAX_ITEMS 65535   // items per call: the grid's y extent
// kind and dtype of b200unet_overlap_operand; field order of that struct
enum OverlapOperandKind { OV_KIND_ONEHOT = 0, OV_KIND_LABEL = 1, OV_KIND_THRESHOLD = 2, OV_KIND_ARGMAX = 3 };
enum OverlapDtype { OV_DTYPE_U8 = 0, OV_DTYPE_I64 = 1, OV_DTYPE_F32 = 2 };
// the (kind, dtype) pairs the kernel reads
enum OverlapForm { OV_ONEHOT_U8 = 0, OV_ONEHOT_F32 = 1, OV_LABEL_U8 = 2, OV_LABEL_I64 = 3, OV_THRESH_F32 = 4, OV_ARGMAX_F32 = 5 };
struct OverlapOperand {
  const void* data;
  int kind, dtype;
  float thr;
};
// counts DEVICE int64 [B][C][3] = (P, G, I), overwritten
int launch_overlap_counts(const OverlapOperand& pred, const OverlapOperand& gt, int B, int C, int D, int H, int W, int64_t* counts,
                          cudaStream_t st);

// ---- tensor-core implicit-GEMM convolution (igemm_conv.cu)
struct ConvSrc {
  Act x;               // A operand (NDHWC bf16, hi[/lo])
  const bf16* w_hi;    // packed weights [T][Cop][Cip] (K = Cip contiguous)
  const bf16* w_lo;    // nullptr in single-pass mode
  int ksz;             // 1 or 3 (2 with nopad: the kernel = stride = 2 case of MONAI's UnetUpBlock transposed convolution)
  int nopad;           // 0: padding = ksz / 2 (resnet.py:12-22); 1: no padding
  int stride;          // 1 or 2 (spatial traversal stride on x)
  int Cip;             // packed K extent of the weights (>= x.C, multiple of 8)
};

struct ConvOp {
  ConvSrc src[2];
  int nsrc;            // 1, or 2 to accumulate a second (1x1x1) source into the same output tile
  int Cop;             // packed weight rows (>= out.C)
  Act out;             // output view (may be a channel slice of a wider buffer)
  const Act* res;      // optional residual added before scale
  const float* scale;  // optional [N][out.C] per-(n,c) multiplier (Dropout3d mask)
  double* stats;       // optional [N][stats_ld][2] per-channel (sum, sumsq) of the stored output
  int stats_ld;
  int mode;            // 0: out = (acc + res) * scale ; 1: GroupNorm/ReLU backward epilogue
  const Act* gn_x;     // mode 1: raw input of the norm (same shape as out)
  const float* coef;   // mode 1: [N][coef_ld][4] (A, B, mu, rstd)
  int coef_ld;
  float slope;         // mode 1: negative slope of the activation (0 = ReLU)
  double* bstats;      // mode 1: [N][coef_ld][2] += (sum dz, sum dz*xhat)
  const float* bias;   // mode 0: optional per-channel bias
  int zero_last;       // mode 0: output voxels on the high boundary of each axis are forced to 0
  int max_ctas;        // > 0: at most this many CTAs per N tile on the persistent halo kernel (diagnostics: several tiles per CTA)
  int tile128;         // != 0: per-tap tiles stay at 128 voxels where 256 would be taken (diagnostics: the one-warpgroup reference)
  int cls_mode;        // 2: ConvTranspose3d(kernel = stride = 2) forward: src[0].x = input at half the output extent, src[0].w = the
                       // PACK_T_FWD pack [8][Cop][Cip]; class p = one tap.  1: data gradient of a 3x3x3 stride-2 padding-1 convolution WITHOUT zero insertion: src[0].x = dY (low
                       // resolution), src[0].w = the flipped data-gradient pack, out = dX at twice the extent; eight
                       // parity-class implicit GEMMs (27 tap products in total instead of 8 x 27) in one launch
};

// The kernel a convolution runs on, decided from the op alone (no device or driver call): launch_igemm_conv launches exactly this.
enum ConvKind { CONV_KIND_TAP = 0, CONV_KIND_HALO = 1, CONV_KIND_CLASS1 = 2, CONV_KIND_CLASS2 = 3, CONV_KIND_HALO_PAIR = 4 };
struct ConvRoute {
  int kind;                 // ConvKind
  int BN, KC;
  int kchunks[2];           // K chunks of KC channels per source
  int npass;                // 1 bf16, 3 split precision
  int cls_pair;             // class mode, bf16: the two W-parity classes share one staging tile and store
  int tw, th, td;           // output voxel tile (class mode: of one parity class, on the source grid)
  int tiles_w, tiles_h, tiles_d;
  int grid[3];
  int stages, blocks_per_sm, smem_bytes;   // ConvCfg of the instantiation
  int wgs;                  // consumer warpgroups per CTA (2: the 256-voxel per-tap tile and the two-plane halo mode)
};
// on a device with num_sms SMs; validates the op: OK or the error launch_igemm_conv would return
int conv_route(const ConvOp& op, int num_sms, ConvRoute* r);
int launch_igemm_conv(const ConvOp& op, cudaStream_t st);

// ---- tensor-core weight gradient (wgrad.cu):  dW[t][ci][co] += sum_v dy[v][co] * a[v*stride + t - pad][ci]
struct WgradOp {
  Act a;       // conv input (normalised activation), NDHWC
  Act dy;      // gradient of the conv output, NDHWC (dims = conv output dims)
  int ksz;     // 1 or 3 (2 with nopad)
  int stride;  // 1 or 2
  int nopad;   // 0: padding = ksz / 2; 1: no padding
  int Cip;     // pitch of the [T][Cip][Cop] fp32 accumulator rows
  int Cop;
  float* dw;   // fp32 [T][Cip][Cop]; accumulated with atomics, caller zero-fills
  // deterministic mode (optional): the split-K CTAs store their partial sums into slots part[slot][T][Cip][Cop] instead of
  // accumulating into dw with atomics; launch_wgrad_reduce then sums the slots in a fixed order.
  float* part;
  size_t part_bytes;
  int* part_splits;   // out: number of slots written
};
int launch_wgrad_reduce(const float* part, int splits, long long elems, float* dw, cudaStream_t st);   // dw = sum_s part[s]
// worst-case bytes of the partial buffer for this shape on a device with num_sms SMs (host-only shape logic)
size_t wgrad_partial_bytes(const WgradOp& op, int num_sms);
// The kernel a weight gradient runs on for a device with num_sms SMs (op.part set: deterministic mode), from the op alone.
enum WgradKind { WGRAD_KIND_SIMT = 0, WGRAD_KIND_TAP = 1, WGRAD_KIND_HALO = 2 };
struct WgradRoute {
  int kind;                 // WgradKind
  int ci8;                  // SIMT: input channels / 8
  int CB, BN, QT;           // tensor-core kernels: channels per M box, N tile, M tiles per CTA (per work item)
  int nci, units, qtiles;   // CB chunks per tap, (tap, chunk) units, M tiles in total
  int groups, cotiles, kblocks, splits, npass;
  int tw, th, td;
  size_t part_bytes;        // deterministic mode: splits * T * Cip * Cop * 4, the partial buffer this launch fills
  int ctas;                 // tensor-core kernels: CTAs of the launch
};
int wgrad_route(const WgradOp& op, int num_sms, WgradRoute* r);
int launch_wgrad(const WgradOp& op, cudaStream_t st);              // dispatcher: SIMT register tile for narrow 1x1x1
bool wgrad_1x1_narrow_eligible(const WgradOp& op);              // 1x1x1, <= 16 input channels: SIMT register tile
int launch_wgrad_1x1_narrow(const WgradOp& op, cudaStream_t st);

}  // namespace b200
