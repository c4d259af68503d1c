// The steps immediately before and after the U-Net path, on the device (HBM-bound, NCDHW at the reference-facing
// boundary).  Paths relative to /root/reference.
//
//   tiles_*        sliding-window inference (monai.inferers.SlidingWindowInferer as called by
//                  unet3d/predict/volumetric.py:147-148, unet3d/train/training_utils.py:106-107): gather a batch of
//                  tiles out of the volume, importance-weighted accumulation of the tile predictions, normalisation
//   one_hot        label map -> one-hot uint8 target (unet3d/utils/one_hot.py:7-37)
//   zscore_*       monai NormalizeIntensity as configured by unet3d/datasets/segmentation.py:77-87 ("zero_mean")
//   label_map      activation + threshold -> label map (unet3d/utils/one_hot.py:46-118)
#include "kernels.h"

namespace b200 {

// ------------------------------------------------------------------------------------------------ sliding window
struct TileList {
  int n;
  int start[B200_MAX_TILES][4];   // (sample, d0, h0, w0)
};

// tiles[b][c][d][h][w] = vol[start[b].n][c][d0+d][h0+h][w0+w]; 4 voxels along w per thread when aligned
__global__ void k_tiles_gather(const float* __restrict__ vol, int C, int D, int H, int W, TileList tl, int rd, int rh, int rw,
                               float* __restrict__ tiles) {
  const long long per = (long long)C * rd * rh * rw;
  const long long total = per * tl.n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int w = (int)(r % rw); r /= rw;
    const int h = (int)(r % rh); r /= rh;
    const int d = (int)(r % rd); r /= rd;
    const int c = (int)(r % C);
    const int b = (int)(r / C);
    const int* s = tl.start[b];
    tiles[i] = __ldg(vol + ((((long long)s[0] * C + c) * D + s[1] + d) * H + s[2] + h) * W + s[3] + w);
  }
}

// Gather formulation (deterministic, no atomics): one thread per voxel of the bounding box of this batch's tiles adds,
// in tile order, every tile prediction that covers it:  out[n][c][v] += pred[b][c][v - start_b] * imp[v - start_b].
__global__ void k_tiles_scatter(const float* __restrict__ pred, int C, TileList tl, int rd, int rh, int rw,
                                const float* __restrict__ imp, float* __restrict__ out, int N, int D, int H, int W, int bd0,
                                int bh0, int bw0, int bd, int bh, int bw) {
  const long long box = (long long)bd * bh * bw;
  const long long total = box * C * N;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int w = bw0 + (int)(r % bw); r /= bw;
    const int h = bh0 + (int)(r % bh); r /= bh;
    const int d = bd0 + (int)(r % bd); r /= bd;
    const int c = (int)(r % C);
    const int n = (int)(r / C);
    float acc = 0.f;
    bool hit = false;
    for (int b = 0; b < tl.n; ++b) {
      const int* s = tl.start[b];
      const int ld = d - s[1], lh = h - s[2], lw = w - s[3];
      if (s[0] == n && ld >= 0 && ld < rd && lh >= 0 && lh < rh && lw >= 0 && lw < rw) {
        const long long lp = ((long long)ld * rh + lh) * rw + lw;
        acc += pred[((long long)b * C + c) * rd * rh * rw + lp] * __ldg(imp + lp);
        hit = true;
      }
    }
    if (hit) {
      float* o = out + ((((long long)n * C + c) * D + d) * H + h) * W + w;
      *o += acc;
    }
  }
}

// cnt[d][h][w] = sum over ALL windows (d0,h0,w0) of the separable scan of imp[v - start]; one thread per voxel
__global__ void k_tiles_count(const int* __restrict__ sd, int nd, const int* __restrict__ sh, int nh, const int* __restrict__ sw,
                              int nw, int rd, int rh, int rw, const float* __restrict__ imp, float* __restrict__ cnt, int D,
                              int H, int W) {
  const long long total = (long long)D * H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int w = (int)(r % W); r /= W;
    const int h = (int)(r % H);
    const int d = (int)(r / H);
    float acc = 0.f;
    for (int a = 0; a < nd; ++a) {
      const int ld = d - sd[a];
      if (ld < 0 || ld >= rd) continue;
      for (int b = 0; b < nh; ++b) {
        const int lh = h - sh[b];
        if (lh < 0 || lh >= rh) continue;
        for (int c = 0; c < nw; ++c) {
          const int lw = w - sw[c];
          if (lw < 0 || lw >= rw) continue;
          acc += __ldg(imp + ((long long)ld * rh + lh) * rw + lw);
        }
      }
    }
    cnt[i] = acc;
  }
}

// out[nc][v] /= cnt[v]
__global__ void k_tiles_normalize(float* __restrict__ out, const float* __restrict__ cnt, long long S, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    out[i] = out[i] / __ldg(cnt + (i % S));
}

static int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  const long long cap = 132LL * 16;
  return (int)(g < 1 ? 1 : g > cap ? cap : g);
}

static int make_tile_list(const int32_t* starts, int n, TileList* tl) {
  B200_REQUIRE(starts && n >= 1 && n <= B200_MAX_TILES, E_INVALID, "tiles: 1..%d tiles per call, got %d", B200_MAX_TILES, n);
  tl->n = n;
  for (int b = 0; b < n; ++b)
    for (int k = 0; k < 4; ++k) tl->start[b][k] = starts[b * 4 + k];
  return OK;
}

int launch_tiles_gather(const float* vol, int N, int C, int D, int H, int W, const int32_t* starts, int ntiles, int rd, int rh,
                        int rw, float* tiles, cudaStream_t st) {
  TileList tl;
  B200_TRY(make_tile_list(starts, ntiles, &tl));
  for (int b = 0; b < ntiles; ++b)
    B200_REQUIRE(tl.start[b][0] >= 0 && tl.start[b][0] < N && tl.start[b][1] >= 0 && tl.start[b][1] + rd <= D && tl.start[b][2] >= 0 &&
                     tl.start[b][2] + rh <= H && tl.start[b][3] >= 0 && tl.start[b][3] + rw <= W,
                 E_INVALID, "tiles_gather: tile %d lies outside the volume", b);
  const long long total = (long long)ntiles * C * rd * rh * rw;
  k_tiles_gather<<<grid_for(total, 256), 256, 0, st>>>(vol, C, D, H, W, tl, rd, rh, rw, tiles);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

int launch_tiles_scatter(const float* pred, int C, const int32_t* starts, int ntiles, int rd, int rh, int rw, const float* imp,
                         float* out, int N, int D, int H, int W, cudaStream_t st) {
  TileList tl;
  B200_TRY(make_tile_list(starts, ntiles, &tl));
  int lo[3] = {D, H, W}, hi[3] = {0, 0, 0};
  const int ext[3] = {rd, rh, rw};
  for (int b = 0; b < ntiles; ++b)
    for (int k = 0; k < 3; ++k) {
      if (tl.start[b][k + 1] < lo[k]) lo[k] = tl.start[b][k + 1];
      if (tl.start[b][k + 1] + ext[k] > hi[k]) hi[k] = tl.start[b][k + 1] + ext[k];
    }
  B200_REQUIRE(lo[0] >= 0 && lo[1] >= 0 && lo[2] >= 0 && hi[0] <= D && hi[1] <= H && hi[2] <= W, E_INVALID,
               "tiles_scatter: a tile lies outside the volume");
  const long long total = (long long)N * C * (hi[0] - lo[0]) * (hi[1] - lo[1]) * (hi[2] - lo[2]);
  k_tiles_scatter<<<grid_for(total, 256), 256, 0, st>>>(pred, C, tl, rd, rh, rw, imp, out, N, D, H, W, lo[0], lo[1], lo[2],
                                                         hi[0] - lo[0], hi[1] - lo[1], hi[2] - lo[2]);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

int launch_tiles_count(const int32_t* sd_dev, int nd, const int32_t* sh_dev, int nh, const int32_t* sw_dev, int nw, int rd, int rh,
                       int rw, const float* imp, float* cnt, int D, int H, int W, cudaStream_t st) {
  B200_REQUIRE(sd_dev && sh_dev && sw_dev && imp && cnt && nd > 0 && nh > 0 && nw > 0, E_INVALID, "tiles_count: bad argument");
  k_tiles_count<<<grid_for((long long)D * H * W, 256), 256, 0, st>>>(sd_dev, nd, sh_dev, nh, sw_dev, nw, rd, rh, rw, imp, cnt, D, H, W);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

int launch_tiles_normalize(float* out, const float* cnt, int NC, long long S, cudaStream_t st) {
  const long long total = (long long)NC * S;
  k_tiles_normalize<<<grid_for(total, 256), 256, 0, st>>>(out, cnt, S, total);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// ------------------------------------------------------------------------------------------------ one-hot target
struct LabelTable {
  int n_channels;
  int begin[B200_MAX_LABEL_CHANNELS + 1];   // channel c owns values[begin[c] .. begin[c+1])
  float values[B200_MAX_LABEL_VALUES];
};

// unet3d/utils/one_hot.py:7-37: data rounded (torch.round: half to even), channel c = 1 where isclose(data, label)
// (atol 1e-8, rtol 1e-5: one_hot.py:40-43) for any label of the channel's group.  data [N][1][S] fp32 -> y [N][L][S] uint8
__global__ void k_one_hot(const float* __restrict__ data, long long S, int N, LabelTable lt, int do_round, uint8_t* __restrict__ y) {
  const long long total = (long long)N * S;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / S, v = i % S;
    float x = data[i];
    if (do_round) x = rintf(x);
    for (int c = 0; c < lt.n_channels; ++c) {
      uint8_t on = 0;
      for (int k = lt.begin[c]; k < lt.begin[c + 1]; ++k) {
        const float lab = lt.values[k];
        if (fabsf(x - lab) <= 1e-8f + 1e-5f * fabsf(lab)) on = 1;
      }
      y[(n * lt.n_channels + c) * S + v] = on;
    }
  }
}

int launch_one_hot(const float* data, int N, long long S, const float* values, const int32_t* begin, int n_channels, int do_round,
                   uint8_t* y, cudaStream_t st) {
  B200_REQUIRE(data && y && values && begin, E_INVALID, "one_hot: null argument");
  B200_REQUIRE(n_channels >= 1 && n_channels <= B200_MAX_LABEL_CHANNELS, E_UNSUPPORTED, "one_hot: 1..%d channels", B200_MAX_LABEL_CHANNELS);
  B200_REQUIRE(begin[0] == 0 && begin[n_channels] <= B200_MAX_LABEL_VALUES, E_UNSUPPORTED, "one_hot: at most %d label values",
               B200_MAX_LABEL_VALUES);
  LabelTable lt;
  lt.n_channels = n_channels;
  for (int c = 0; c <= n_channels; ++c) lt.begin[c] = begin[c];
  for (int k = 0; k < begin[n_channels]; ++k) lt.values[k] = values[k];
  k_one_hot<<<grid_for((long long)N * S, 256), 256, 0, st>>>(data, S, N, lt, do_round, y);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// ------------------------------------------------------------------------------------------------ z-score
// monai.transforms.NormalizeIntensity(nonzero, channel_wise): (x - mean) / std over the selected voxels (population std,
// std == 0 -> 1); with nonzero only the non-zero voxels contribute and are changed.  x [G][S] fp32, one group per
// normalisation unit (G = C when channel_wise, else 1 with S = C * voxels).
__global__ void k_zscore_stats(const float* __restrict__ x, long long S, int nonzero, double* __restrict__ stats) {
  __shared__ double sh[3][32];
  const float* p = x + (long long)blockIdx.y * S;
  double s = 0, q = 0, k = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < S; i += (long long)gridDim.x * blockDim.x) {
    const float v = p[i];
    if (!nonzero || v != 0.f) { s += v; q += (double)v * v; k += 1; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); k += __shfl_xor_sync(0xffffffffu, k, o);
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { sh[0][w] = s; sh[1][w] = q; sh[2][w] = k; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double ts = 0, tq = 0, tk = 0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { ts += sh[0][i]; tq += sh[1][i]; tk += sh[2][i]; }
    atomicAdd(&stats[blockIdx.y * 3 + 0], ts);
    atomicAdd(&stats[blockIdx.y * 3 + 1], tq);
    atomicAdd(&stats[blockIdx.y * 3 + 2], tk);
  }
}

__global__ void k_zscore_apply(const float* __restrict__ x, long long S, int nonzero, const double* __restrict__ stats,
                               float* __restrict__ y) {
  const double cnt = stats[blockIdx.y * 3 + 2];
  const double mean = cnt > 0 ? stats[blockIdx.y * 3] / cnt : 0.0;
  double var = cnt > 0 ? stats[blockIdx.y * 3 + 1] / cnt - mean * mean : 0.0;
  if (var < 0) var = 0;
  double sd = sqrt(var);
  if (sd == 0.0) sd = 1.0;
  const float m = (float)mean, inv = (float)(1.0 / sd);
  const float* p = x + (long long)blockIdx.y * S;
  float* o = y + (long long)blockIdx.y * S;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < S; i += (long long)gridDim.x * blockDim.x) {
    const float v = p[i];
    o[i] = (!nonzero || v != 0.f) ? (v - m) * inv : v;
  }
}

int launch_zscore(const float* x, int groups, long long S, int nonzero, double* stats, float* y, cudaStream_t st) {
  B200_REQUIRE(x && y && stats && groups > 0 && S > 0, E_INVALID, "zscore: bad argument");
  B200_CHECK_CUDA(cudaMemsetAsync(stats, 0, sizeof(double) * 3 * groups, st));
  int chunks = (132 * 8 + groups - 1) / groups;
  const long long per = (S + 1023) / 1024;
  if (chunks > per) chunks = (int)(per < 1 ? 1 : per);
  k_zscore_stats<<<dim3(chunks, groups), 256, 0, st>>>(x, S, nonzero, stats);
  B200_CHECK_CUDA(cudaGetLastError());
  k_zscore_apply<<<dim3(chunks, groups), 256, 0, st>>>(x, S, nonzero, stats, y);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

// ------------------------------------------------------------------------------------------------ label map
// unet3d/utils/one_hot.py:46-118 on one sample: p [L][S] (logits when act != 0) -> int16 label map [S].
//   hierarchy (one_hot.py:92-110):  roi_k = AND_{i<=k} (p_i > thr);  label_map[roi_k] = labels[k]
//   otherwise (one_hot.py:64-89):   mask = any_i (p_i > thr)  |  sum_i p_i > thr;  label = labels[argmax_i p_i] where mask
// act: 0 none, 1 sigmoid, 2 softmax over the L channels (volumetric.py:151-156 applied first).
struct LabelMapArgs {
  int L;
  int16_t labels[B200_MAX_LABEL_CHANNELS];
};

// Two passes over the channels and no per-thread array of L values (L goes up to 128): the first gives the maximum and the
// softmax denominator, the second recomputes each activated value with the same float expression and folds it in channel order.
__global__ void k_label_map(const float* __restrict__ p, long long S, LabelMapArgs a, int act, float thr, int hierarchy,
                            int sum_then_threshold, int16_t* __restrict__ out) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < S; v += (long long)gridDim.x * blockDim.x) {
    float mx = -INFINITY, den = 0.f;
    for (int c = 0; c < a.L; ++c) mx = fmaxf(mx, p[(long long)c * S + v]);
    if (act == 2)
      for (int c = 0; c < a.L; ++c) den += expf(p[(long long)c * S + v] - mx);
    auto q = [&](int c) -> float {
      const float x = p[(long long)c * S + v];
      if (act == 1) return 1.f / (1.f + expf(-x));
      if (act == 2) return expf(x - mx) / den;
      return x;
    };
    int16_t lab = 0;
    if (hierarchy) {
      bool roi = true;
      for (int c = 0; c < a.L; ++c) {
        roi = roi && (q(c) > thr);
        if (roi) lab = a.labels[c];
      }
    } else {
      bool mask = false;
      float sum = 0.f, best = q(0);
      int arg = 0;
      for (int c = 0; c < a.L; ++c) {
        const float qc = q(c);
        mask = mask || (qc > thr);
        sum += qc;
        if (qc > best) { best = qc; arg = c; }   // torch.argmax: first maximal index
      }
      if (sum_then_threshold) mask = sum > thr;
      if (mask) lab = a.labels[arg];
    }
    out[v] = lab;
  }
}

int launch_label_map(const float* p, int L, long long S, const int32_t* labels, int act, float thr, int hierarchy,
                     int sum_then_threshold, int16_t* out, cudaStream_t st) {
  B200_REQUIRE(p && out && labels, E_INVALID, "label_map: null argument");
  B200_REQUIRE(L >= 1 && L <= B200_MAX_LABEL_CHANNELS, E_UNSUPPORTED, "label_map: 1..%d channels", B200_MAX_LABEL_CHANNELS);
  LabelMapArgs a;
  a.L = L;
  for (int c = 0; c < L; ++c) a.labels[c] = (int16_t)labels[c];
  k_label_map<<<grid_for(S, 256), 256, 0, st>>>(p, S, a, act, thr, hierarchy, sum_then_threshold, out);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

}  // namespace b200
