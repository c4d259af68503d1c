// Connected-component labelling of binary 3D masks on the device, and the ranking of the components by size: the
// clean-up after a segmentation (SimpleITK ConnectedComponent + RelabelComponent(sortByObjectSize=True), MONAI's
// KeepLargestConnectedComponent), without copying the prediction to the host.
//
// Block-based union-find with atomicMin (Playne & Hawick 2018; the tile-local step follows Allegretti, Bolelli & Grana 2019).
// Every union links the larger root under the smaller one, so a component's root is its minimum linear index and the raster
// numbering of scipy.ndimage.label is a prefix sum over root flags.  Labels are exact integers, independent of scheduling.
//
//   k_cc_local    one 4x8x32 tile per block: union-find in shared memory over the backward neighbours inside the tile;
//                 writes parent = the voxel's tile root (global linear index), -1 for background
//   k_cc_merge    tile-border voxels: atomicMin union with their backward neighbours in other tiles (faces, and for 18/26
//                 connectivity the edge and corner neighbours in diagonal tiles)
//   k_cc_flatten  parent = root (path halving), flag = voxel is a root
//   scan          per volume, inclusive sum of the flags: rank of each root in raster order
//   k_cc_raster   label = rank[root]; counts[v] = K_v
//   k_cc_count    sizes[v][label - 1] (warp-aggregated integer atomics: exact)
//   sort_by_size  per volume: keys (S - size, label) radix-sorted ascending -> new label = position + 1; one rewrite pass
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "kernels.h"

namespace b200 {
namespace {

constexpr int TD = 4, TH = 8, TW = 32, TV = TD * TH * TW;

// backward neighbours (dz, dy, dx): the offsets before the voxel in raster order.  The first 3 / 9 / 13 are those of the 6- /
// 18- / 26-neighbourhood (connectivity 1 / 2 / 3).
__constant__ int8_t c_off[13][3] = {{-1, 0, 0},  {0, -1, 0},  {0, 0, -1},  {-1, -1, 0}, {-1, 1, 0},
                                    {-1, 0, -1}, {-1, 0, 1},  {0, -1, -1}, {0, -1, 1},  {-1, -1, -1},
                                    {-1, -1, 1}, {-1, 1, -1}, {-1, 1, 1}};

struct Geo {
  int D, H, W, S;   // S = D * H * W < 2^31
  int tH, tW;       // tiles along H and W
  int tiles;        // tiles per volume
};

struct TileCoord {
  long long base;   // v * S
  int lx, ly, lz, x0, y0, z0, x, y, z;
  bool in;
};

__device__ __forceinline__ TileCoord tile_coord(const Geo& g) {
  TileCoord c;
  const long long blk = blockIdx.x;
  const int v = (int)(blk / g.tiles);
  int t = (int)(blk % g.tiles);
  c.x0 = (t % g.tW) * TW; t /= g.tW;
  c.y0 = (t % g.tH) * TH;
  c.z0 = (t / g.tH) * TD;
  c.lx = threadIdx.x % TW; c.ly = (threadIdx.x / TW) % TH; c.lz = threadIdx.x / (TW * TH);
  c.x = c.x0 + c.lx; c.y = c.y0 + c.ly; c.z = c.z0 + c.lz;
  c.in = c.x < g.W && c.y < g.H && c.z < g.D;
  c.base = (long long)v * g.S;
  return c;
}

__device__ __forceinline__ int find_shared(const volatile int* p, int a) {
  int q = p[a];
  while (q != a) { a = q; q = p[a]; }
  return a;
}

// parents only decrease and every root is its set's minimum; a failed atomicMin means b gained a parent: retry from there
__device__ void union_shared(int* p, int a, int b) {
  while (true) {
    a = find_shared(p, a);
    b = find_shared(p, b);
    if (a == b) return;
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(p + b, a);
    if (old == b) return;
    b = old;
  }
}

// global parents are read through L2 (__ldcg): other blocks link roots concurrently
__device__ __forceinline__ int find_global(const int32_t* p, int a) {
  int q = __ldcg(p + a);
  while (q != a) { a = q; q = __ldcg(p + a); }
  return a;
}

__device__ void union_global(int32_t* p, int a, int b) {
  while (true) {
    a = find_global(p, a);
    b = find_global(p, b);
    if (a == b) return;
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(p + b, a);
    if (old == b) return;
    b = old;
  }
}

__global__ void __launch_bounds__(TV) k_cc_local(const uint8_t* __restrict__ mask, Geo g, int nb, int32_t* __restrict__ P) {
  __shared__ int s[TV];
  const TileCoord c = tile_coord(g);
  const int t = threadIdx.x;
  const int i = c.in ? (c.z * g.H + c.y) * g.W + c.x : 0;
  const bool fg = c.in && mask[c.base + i] != 0;
  s[t] = fg ? t : -1;
  __syncthreads();
  if (fg) {
    for (int k = 0; k < nb; ++k) {
      const int az = c.lz + c_off[k][0], ay = c.ly + c_off[k][1], ax = c.lx + c_off[k][2];
      if (az < 0 || ay < 0 || ay >= TH || ax < 0 || ax >= TW) continue;   // az <= lz < TD
      const int j = (az * TH + ay) * TW + ax;
      if (s[j] >= 0) union_shared(s, t, j);                               // background entries stay -1
    }
  }
  __syncthreads();
  if (c.in) {
    int r = -1;
    if (fg) {
      const int q = find_shared(s, t);
      r = ((c.z0 + q / (TW * TH)) * g.H + c.y0 + (q / TW) % TH) * g.W + c.x0 + q % TW;
    }
    P[c.base + i] = r;
  }
}

__global__ void __launch_bounds__(TV) k_cc_merge(Geo g, int nb, int32_t* __restrict__ P) {
  const TileCoord c = tile_coord(g);
  if (!c.in) return;
  if (c.lz > 0 && c.ly > 0 && c.ly < TH - 1 && c.lx > 0 && c.lx < TW - 1) return;   // every backward neighbour is in the tile
  int32_t* p = P + c.base;
  const int i = (c.z * g.H + c.y) * g.W + c.x;
  if (__ldcg(p + i) < 0) return;
  for (int k = 0; k < nb; ++k) {
    const int dz = c_off[k][0], dy = c_off[k][1], dx = c_off[k][2];
    const int az = c.lz + dz, ay = c.ly + dy, ax = c.lx + dx;
    if (az >= 0 && ay >= 0 && ay < TH && ax >= 0 && ax < TW) continue;     // same tile: done by k_cc_local
    const int nz = c.z + dz, ny = c.y + dy, nx = c.x + dx;
    if (nz < 0 || ny < 0 || ny >= g.H || nx < 0 || nx >= g.W) continue;
    const int j = (nz * g.H + ny) * g.W + nx;
    if (__ldcg(p + j) >= 0) union_global(p, i, j);
  }
}

// No unions run here: every parent is an ancestor at any moment, so concurrent path halving is safe.  The halving store is an
// atomicMin: another thread may already have written the root (its set's minimum) into that voxel, and a plain store of the
// grandparent would undo it.
__global__ void k_cc_flatten(int32_t* __restrict__ P, int32_t* __restrict__ flag, long long total, int S) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int a = P[e];
    if (a < 0) { flag[e] = 0; continue; }
    const long long base = e - e % S;
    int32_t* p = P + base;
    int x = a;
    while (true) {
      const int px = __ldcg(p + x);
      if (px == x) break;
      const int gx = __ldcg(p + px);
      if (gx == px) { x = px; break; }
      atomicMin(p + x, gx);
      x = gx;
    }
    P[e] = x;
    flag[e] = x == (int)(e - base);
  }
}

__global__ void k_cc_raster(int32_t* __restrict__ L, const int32_t* __restrict__ rank, long long total, int S,
                            int32_t* __restrict__ counts) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long base = e - e % S;
    const int a = L[e];
    L[e] = a < 0 ? 0 : rank[base + a];
    if (e - base == S - 1) counts[e / S] = rank[e];
  }
}

// sizes[v][label - 1] += 1; lanes of a warp holding the same label add once (a large component would otherwise serialise
// millions of atomics on one address).  The loop bound is warp-uniform, so every lane takes part in __match_any_sync.
__global__ void k_cc_count(const int32_t* __restrict__ L, int32_t* __restrict__ sizes, long long total, int S) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long e0 = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31); e0 < total; e0 += stride) {
    const long long e = e0 + lane;
    const int lab = e < total ? L[e] : 0;
    const long long key = lab > 0 ? e - e % S + lab - 1 : -1;
    const unsigned same = __match_any_sync(0xffffffffu, (unsigned long long)key);
    if (lab > 0 && lane == __ffs(same) - 1) atomicAdd(sizes + key, __popc(same));
  }
}

// key = (S - size) << 32 | label - 1: ascending order = size descending, ties by raster label; sizes of 0 (labels beyond K_v)
// give S << 32 and sort last
__global__ void k_cc_keys(const int32_t* __restrict__ sizes, int n, int S, uint64_t* __restrict__ keys) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x)
    keys[j] = ((uint64_t)(S - sizes[j]) << 32) | (uint32_t)j;
}

// newlab[label - 1] = position + 1 (written over the sizes, which the keys already hold)
__global__ void k_cc_perm(const uint64_t* __restrict__ sorted, int n, int S, int32_t* __restrict__ newlab) {
  for (int pos = blockIdx.x * blockDim.x + threadIdx.x; pos < n; pos += gridDim.x * blockDim.x) {
    const uint64_t k = sorted[pos];
    if ((int)(k >> 32) < S) newlab[(uint32_t)k] = pos + 1;
  }
}

__global__ void k_cc_relabel(int32_t* __restrict__ L, const int32_t* __restrict__ newlab, long long total, int S) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int a = L[e];
    if (a > 0) L[e] = newlab[e - e % S + a - 1];
  }
}

int grid_for(long long total, int block) {
  const long long g = (total + block - 1) / block, cap = 132LL * 16;
  return (int)(g < 1 ? 1 : g > cap ? cap : g);
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// Scratch: work int32 [nvol][S] (ranks, then sizes, then the size-order map), two uint64 key buffers of kmax entries (one
// volume is sorted at a time), and CUB's temporary storage for a scan of S and a sort of kmax items.  kmax = ceil(S / 2) is
// the largest component count of any connectivity (the 6-connected checkerboard).
struct Layout {
  size_t work, keys, temp, total;
  int kmax;
};

int check_shape(int nvol, int d, int h, int w, Geo* g) {
  B200_REQUIRE(nvol >= 1 && d >= 1 && h >= 1 && w >= 1, E_INVALID, "cc: nvol, d, h, w must be >= 1 (got %d, %d, %d, %d)", nvol, d,
               h, w);
  const long long S = (long long)d * h * w;
  B200_REQUIRE(S < (1LL << 31), E_UNSUPPORTED, "cc: d*h*w = %lld voxels per volume; at most 2^31 - 1", S);
  g->D = d; g->H = h; g->W = w; g->S = (int)S;
  g->tH = ceil_div(h, TH); g->tW = ceil_div(w, TW);
  const long long tiles = (long long)ceil_div(d, TD) * g->tH * g->tW;
  B200_REQUIRE(tiles * nvol < (1LL << 31), E_UNSUPPORTED, "cc: %d volumes of %lld tiles exceed one launch grid", nvol, tiles);
  g->tiles = (int)tiles;
  return OK;
}

int layout(int nvol, const Geo& g, Layout* L) {
  L->kmax = (int)(((long long)g.S + 1) / 2);
  size_t scan_b = 0, sort_b = 0;
  B200_CHECK_CUDA(cub::DeviceScan::InclusiveSum(nullptr, scan_b, (int32_t*)nullptr, (int32_t*)nullptr, g.S));
  cub::DoubleBuffer<uint64_t> db(nullptr, nullptr);
  B200_CHECK_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, sort_b, db, L->kmax, 0, 64));
  L->work = align256(sizeof(int32_t) * (size_t)nvol * g.S);
  L->keys = align256(sizeof(uint64_t) * (size_t)L->kmax);
  L->temp = align256(scan_b > sort_b ? scan_b : sort_b);
  L->total = L->work + 2 * L->keys + L->temp;
  return OK;
}

}  // namespace

size_t cc_scratch_bytes(int nvol, int d, int h, int w) {
  Geo g;
  Layout L;
  if (check_shape(nvol, d, h, w, &g) != OK || layout(nvol, g, &L) != OK) return 0;
  return L.total;
}

int launch_cc_label(const uint8_t* mask, int nvol, int d, int h, int w, int connectivity, int32_t* labels, int32_t* counts,
                    void* scratch, cudaStream_t st) {
  B200_REQUIRE(mask && labels && counts && scratch, E_INVALID, "cc_label: null argument");
  B200_REQUIRE(connectivity >= 1 && connectivity <= 3, E_INVALID, "cc_label: connectivity must be 1, 2 or 3 (got %d)", connectivity);
  Geo g;
  Layout L;
  B200_TRY(check_shape(nvol, d, h, w, &g));
  B200_TRY(layout(nvol, g, &L));
  char* base = static_cast<char*>(scratch);
  int32_t* work = reinterpret_cast<int32_t*>(base);
  void* temp = base + L.work + 2 * L.keys;
  const int nb = connectivity == 1 ? 3 : connectivity == 2 ? 9 : 13;
  const long long total = (long long)nvol * g.S;
  const unsigned blocks = (unsigned)((long long)nvol * g.tiles);

  k_cc_local<<<blocks, TV, 0, st>>>(mask, g, nb, labels);
  B200_CHECK_CUDA(cudaGetLastError());
  k_cc_merge<<<blocks, TV, 0, st>>>(g, nb, labels);
  B200_CHECK_CUDA(cudaGetLastError());
  k_cc_flatten<<<grid_for(total, 256), 256, 0, st>>>(labels, work, total, g.S);
  B200_CHECK_CUDA(cudaGetLastError());
  for (int v = 0; v < nvol; ++v) {
    int32_t* w_v = work + (long long)v * g.S;
    size_t tb = L.temp;
    B200_CHECK_CUDA(cub::DeviceScan::InclusiveSum(temp, tb, w_v, w_v, g.S, st));
  }
  k_cc_raster<<<grid_for(total, 256), 256, 0, st>>>(labels, work, total, g.S, counts);
  B200_CHECK_CUDA(cudaGetLastError());
  B200_CHECK_CUDA(cudaMemsetAsync(work, 0, sizeof(int32_t) * (size_t)total, st));
  k_cc_count<<<grid_for(total, 256), 256, 0, st>>>(labels, work, total, g.S);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

int launch_cc_sort_by_size(int32_t* labels, int nvol, int d, int h, int w, int max_count, void* scratch, cudaStream_t st) {
  B200_REQUIRE(labels && scratch, E_INVALID, "cc_sort_by_size: null argument");
  Geo g;
  Layout L;
  B200_TRY(check_shape(nvol, d, h, w, &g));
  B200_TRY(layout(nvol, g, &L));
  B200_REQUIRE(max_count >= 0 && max_count <= L.kmax, E_INVALID, "cc_sort_by_size: max_count %d outside [0, %d]", max_count, L.kmax);
  if (max_count == 0) return OK;
  char* base = static_cast<char*>(scratch);
  int32_t* work = reinterpret_cast<int32_t*>(base);
  uint64_t* k0 = reinterpret_cast<uint64_t*>(base + L.work);
  uint64_t* k1 = reinterpret_cast<uint64_t*>(base + L.work + L.keys);
  void* temp = base + L.work + 2 * L.keys;
  int end_bit = 32;                                   // the high word is S - size <= S
  while (end_bit < 64 && ((unsigned long long)g.S >> (end_bit - 32)) != 0) ++end_bit;
  for (int v = 0; v < nvol; ++v) {
    int32_t* w_v = work + (long long)v * g.S;
    k_cc_keys<<<grid_for(max_count, 256), 256, 0, st>>>(w_v, max_count, g.S, k0);
    B200_CHECK_CUDA(cudaGetLastError());
    cub::DoubleBuffer<uint64_t> db(k0, k1);
    size_t tb = 0;
    B200_CHECK_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, db, max_count, 0, end_bit, st));
    B200_REQUIRE(tb <= L.temp, E_INVALID, "cc_sort_by_size: sort needs %zu temporary bytes, the layout has %zu", tb, L.temp);
    tb = L.temp;
    B200_CHECK_CUDA(cub::DeviceRadixSort::SortKeys(temp, tb, db, max_count, 0, end_bit, st));
    k_cc_perm<<<grid_for(max_count, 256), 256, 0, st>>>(db.Current(), max_count, g.S, w_v);
    B200_CHECK_CUDA(cudaGetLastError());
  }
  const long long total = (long long)nvol * g.S;
  k_cc_relabel<<<grid_for(total, 256), 256, 0, st>>>(labels, work, total, g.S);
  B200_CHECK_CUDA(cudaGetLastError());
  return OK;
}

}  // namespace b200
