// Sliding-window detection (SlidingWindowInferenceDetectionWrapper, reference:
// training/models/detection_models/sliding_window_detection_forward_wrapper.py:107-166, SG 3.7.1):
//
//   sgb_sliding_window_gather  cuts every tile of a chunk out of the pre-processed bf16 NHWC canvas in one launch (zero outside
//                              the canvas: the reference pads in processed space with torch.zeros, :147-149);
//   sgb_sliding_window_merge   the reference's per-image merge (:118-133): the rows of every tile of an image shifted by the
//                              tile origin (fp32 add, no clipping), concatenated in (tile, row) order, then torchvision's CPU
//                              batched_nms(boxes, conf, label, iou) -- the coordinate trick iff boxes.numel() <= 4000, per-class
//                              NMS otherwise -- for every image of the batch, without a host synchronisation.
//
// Merge schedule (DESIGN.md section 4.9), workspace linear in the candidates (no n x n matrix):
//   1. sw_compact_kernel      one CTA per image: per-tile prefix of the counts, ordered compaction with the origin add, label
//                             histogram -> per-class offsets, max coordinate -> trick offset, 64-bit sort keys (score desc, position);
//   2. sw_sort_*              bitonic sort of each image's keys: 2048-key tiles in shared memory, global passes for larger strides;
//   3. sw_gather_sorted       boxes for NMS (offset under the trick), areas and labels in sorted order;
//   4. sw_merge_nms_kernel    one CTA per (class, image) -- one per image under the trick -- walks the sorted list in blocks of
//                             64 candidates of its class: every candidate of the block is tested against the class's kept list in
//                             parallel, the block is resolved within itself by a 64 x 64 IoU bit matrix and one 64-step sweep,
//                             and the block's survivors are appended to the kept list;
//   5. sw_merge_output_kernel ordered compaction of the kept flags in (score desc, position) order -> rows and counts.
// The result order is (score desc, position asc) in both torchvision paths: the trick's nms returns it, and the per-class path's final
// `scores.sort(descending=True)` agrees with it except among exactly tied scores (DESIGN.md section 4).
#include "common.cuh"
#include "nms_math.cuh"

#include <math.h>

namespace {

constexpr int NT = 1024;
constexpr int SORT_TILE = 2048;  // keys sorted per CTA in shared memory
constexpr int NB = 64;           // candidates resolved per block of the greedy pass
constexpr int KEEP_LANES = NT / NB;
constexpr int MAX_CLASSES = 4096;

struct ImageMeta {
  int n;       // candidates of the image
  int status;  // 0 ok, 1 bad count, 2 bad label
  int trick;   // coordinate-offset path
  float step;  // max_coordinate + 1
};

struct MergeWs {
  float* ox[4];        // [B * cap] boxes in canvas pixels, list order
  float* score;        // [B * cap]
  int* label;          // [B * cap]
  unsigned long long* keys;  // [B * np2]
  float* sbx[4];       // [B * cap] boxes for NMS, sorted order
  float* sarea;        // [B * cap]
  int* slabel;         // [B * cap]
  int* keep;           // [B * cap] sorted order
  float* kbx[5];       // [B * cap] kept lists (x1, y1, x2, y2, area), per class at cls_off
  int* cls_off;        // [B * (ncls + 1)]
  ImageMeta* meta;     // [B]
};

__device__ __forceinline__ int block_exclusive_scan(int v, int* warp_sums, int* total) {
  // 1024 threads; returns the exclusive prefix of v in thread order
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int s = warp_sums[lane];
    int t = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += y;
    }
    warp_sums[lane] = t - s;
    if (lane == 31) *total = t;
  }
  __syncthreads();
  const int r = warp_sums[warp] + x - v;
  __syncthreads();
  return r;
}

// ---------------------------------------------------------------------------------------------------------------- gather
__global__ void sw_gather_kernel(const uint4* __restrict__ canvas, int B, int H, int W, int vec_per_px, const int* __restrict__ tiles, int T,
                                 int tile, uint4* __restrict__ out) {
  const int64_t per_tile = (int64_t)tile * tile * vec_per_px;
  const int64_t total = per_tile * T;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i / per_tile);
    const int64_t r = i - t * per_tile;
    const int v = (int)(r % vec_per_px);
    const int64_t px = r / vec_per_px;
    const int ty = (int)(px / tile), tx = (int)(px - (int64_t)ty * tile);
    const int b = tiles[3 * t], y = tiles[3 * t + 1] + ty, x = tiles[3 * t + 2] + tx;
    uint4 val = make_uint4(0u, 0u, 0u, 0u);
    if (b >= 0 && b < B && y >= 0 && y < H && x >= 0 && x < W) val = canvas[(((int64_t)b * H + y) * W + x) * vec_per_px + v];
    out[i] = val;
  }
}

// ---------------------------------------------------------------------------------------------------------------- merge
__global__ void __launch_bounds__(NT, 1) sw_compact_kernel(const float* __restrict__ rows, const int* __restrict__ counts, const int* __restrict__ tiles,
                                                          const int* __restrict__ image_tiles, int P, int ncls, int cap, int np2, MergeWs w) {
  __shared__ int hist[MAX_CLASSES];
  __shared__ int warp_sums[32];
  __shared__ int s_total, s_status;
  __shared__ float s_max[32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int t0 = image_tiles[b], t1 = image_tiles[b + 1];
  for (int c = tid; c < ncls; c += NT) hist[c] = 0;
  if (tid == 0) s_status = 0;
  __syncthreads();
  int* toff = w.keep + (int64_t)b * cap;  // per-tile offsets of this image (the keep flags are written later, by sw_gather_sorted)
  // per-tile exclusive prefix of the counts, in chunks of NT tiles
  int base = 0;
  for (int c0 = t0; c0 < t1; c0 += NT) {
    const int t = c0 + tid;
    int c = 0;
    if (t < t1) {
      c = counts[t];
      if (c < 0 || c > P) {
        s_status = 1;
        c = 0;
      }
    }
    const int ex = block_exclusive_scan(c, warp_sums, &s_total);
    if (t < t1) toff[t - t0] = base + ex;
    base += s_total;
    __syncthreads();
  }
  const int n = base;
  // ordered compaction: warp w takes tiles w, w + 32, ...; its lanes copy the tile's rows
  float lmax = -INFINITY;
  const int64_t o = (int64_t)b * cap;
  for (int t = t0 + warp; t < t1; t += NT / 32) {
    int c = counts[t];
    c = (c < 0 || c > P) ? 0 : c;
    const int off = toff[t - t0];
    const float y0 = (float)tiles[3 * t + 1], x0 = (float)tiles[3 * t + 2];
    for (int r = lane; r < c; r += 32) {
      const float* row = rows + ((int64_t)t * P + r) * 6;
      const float x1 = sgb_nms::add_rn(row[0], x0), y1 = sgb_nms::add_rn(row[1], y0);
      const float x2 = sgb_nms::add_rn(row[2], x0), y2 = sgb_nms::add_rn(row[3], y0);
      const float lf = row[5];
      const int lab = (int)lf;
      const int j = off + r;
      const bool ok = lab >= 0 && lab < ncls && (float)lab == lf;
      if (!ok) s_status = 2;  // the image is refused; its slot still gets a valid label and key so that the sort stays in bounds
      else atomicAdd(&hist[lab], 1);
      w.ox[0][o + j] = x1;
      w.ox[1][o + j] = y1;
      w.ox[2][o + j] = x2;
      w.ox[3][o + j] = y2;
      w.score[o + j] = row[4];
      w.label[o + j] = ok ? lab : 0;
      w.keys[(int64_t)b * np2 + j] = sgb_nms::sort_key(row[4], (uint32_t)j);
      lmax = fmaxf(lmax, fmaxf(fmaxf(x1, y1), fmaxf(x2, y2)));
    }
  }
  for (int j = n + tid; j < np2; j += NT) w.keys[(int64_t)b * np2 + j] = ~0ull;
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, s));
  if (lane == 0) s_max[warp] = lmax;
  __syncthreads();
  if (tid == 0) {
    float m = -INFINITY;
    for (int i = 0; i < 32; ++i) m = fmaxf(m, s_max[i]);
    int* co = w.cls_off + (int64_t)b * (ncls + 1);
    int acc = 0;
    for (int c = 0; c < ncls; ++c) {
      co[c] = acc;
      acc += hist[c];
    }
    co[ncls] = acc;
    ImageMeta mt;
    mt.n = n;
    mt.status = s_status;
    mt.trick = 4 * (int64_t)n <= 4000 ? 1 : 0;  // torchvision (CPU): coordinate trick iff boxes.numel() <= 4000
    mt.step = sgb_nms::offset_step(m);
    w.meta[b] = mt;
  }
}

// bitonic network over each image's np2 keys (ascending); direction of a pair: ascending iff (index & k) == 0
__global__ void __launch_bounds__(NT) sw_sort_local_kernel(unsigned long long* keys, int np2, int k_first, int k_last) {
  __shared__ unsigned long long s[SORT_TILE];
  unsigned long long* g = keys + (int64_t)blockIdx.y * np2 + (int64_t)blockIdx.x * SORT_TILE;
  const int gbase = blockIdx.x * SORT_TILE;
  for (int i = threadIdx.x; i < SORT_TILE; i += NT) s[i] = g[i];
  __syncthreads();
  for (int k = k_first; k <= k_last; k <<= 1) {
    for (int j = (k <= SORT_TILE ? k : SORT_TILE) >> 1; j > 0; j >>= 1) {
      const int t = threadIdx.x;
      const int i = 2 * j * (t / j) + t % j;  // lower index of this thread's pair
      const int ixj = i + j;
      const bool up = ((gbase + i) & k) == 0;
      const unsigned long long a = s[i], c = s[ixj];
      if ((a > c) == up) {
        s[i] = c;
        s[ixj] = a;
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < SORT_TILE; i += NT) g[i] = s[i];
}

__global__ void sw_sort_global_kernel(unsigned long long* keys, int np2, int k, int j) {
  unsigned long long* g = keys + (int64_t)blockIdx.y * np2;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= np2 / 2) return;
  const int i = 2 * j * (t / j) + t % j;
  const int ixj = i + j;
  const bool up = (i & k) == 0;
  const unsigned long long a = g[i], c = g[ixj];
  if ((a > c) == up) {
    g[i] = c;
    g[ixj] = a;
  }
}

__global__ void sw_gather_sorted_kernel(int cap, int np2, MergeWs w) {
  const int b = blockIdx.y;
  const ImageMeta mt = w.meta[b];
  if (mt.status != 0) return;
  const int64_t o = (int64_t)b * cap;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < mt.n; i += gridDim.x * blockDim.x) {
    const int p = (int)(w.keys[(int64_t)b * np2 + i] & 0xffffffffu);
    const int lab = w.label[o + p];
    float x1 = w.ox[0][o + p], y1 = w.ox[1][o + p], x2 = w.ox[2][o + p], y2 = w.ox[3][o + p];
    if (mt.trick) {
      const float off = sgb_nms::label_offset(lab, mt.step);
      x1 = sgb_nms::add_rn(x1, off);
      y1 = sgb_nms::add_rn(y1, off);
      x2 = sgb_nms::add_rn(x2, off);
      y2 = sgb_nms::add_rn(y2, off);
    }
    w.sbx[0][o + i] = x1;
    w.sbx[1][o + i] = y1;
    w.sbx[2][o + i] = x2;
    w.sbx[3][o + i] = y2;
    w.sarea[o + i] = sgb_nms::area(x1, y1, x2, y2);
    w.slabel[o + i] = lab;
    w.keep[o + i] = 0;
  }
}

__global__ void __launch_bounds__(NT, 1) sw_merge_nms_kernel(int cap, int ncls, double iou_thr, MergeWs w) {
  __shared__ int cidx[NT];
  __shared__ float cb[5][NB];
  __shared__ int sup[NB];
  __shared__ unsigned long long mask[NB];
  __shared__ int warp_sums[32];
  __shared__ int s_total;
  __shared__ unsigned long long s_kmask;
  const int c = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const ImageMeta mt = w.meta[b];
  if (mt.status != 0 || mt.n == 0) return;
  if (mt.trick && c > 0) return;
  const int* co = w.cls_off + (int64_t)b * (ncls + 1);
  if (!mt.trick && co[c + 1] == co[c]) return;
  const int64_t o = (int64_t)b * cap;
  const int64_t kb = o + (mt.trick ? 0 : co[c]);
  int nk = 0;
  for (int base = 0; base < mt.n; base += NT) {
    const int i = base + tid;
    const bool mine = i < mt.n && (mt.trick || w.slabel[o + i] == c);
    const int pos = block_exclusive_scan(mine ? 1 : 0, warp_sums, &s_total);
    const int m = s_total;
    if (mine) cidx[pos] = i;
    __syncthreads();
    for (int s0 = 0; s0 < m; s0 += NB) {
      const int ns = min(NB, m - s0);
      if (tid < ns) {
        const int64_t q = o + cidx[s0 + tid];
        cb[0][tid] = w.sbx[0][q];
        cb[1][tid] = w.sbx[1][q];
        cb[2][tid] = w.sbx[2][q];
        cb[3][tid] = w.sbx[3][q];
        cb[4][tid] = w.sarea[q];
        sup[tid] = 0;
        mask[tid] = 0ull;
      }
      __syncthreads();
      {  // candidates against the kept list: KEEP_LANES threads per candidate stride the list
        const int ci = tid % NB, g = tid / NB;
        if (ci < ns) {
          const float jx1 = cb[0][ci], jy1 = cb[1][ci], jx2 = cb[2][ci], jy2 = cb[3][ci], ja = cb[4][ci];
          for (int k = g; k < nk; k += KEEP_LANES) {
            if (sgb_nms::suppresses(w.kbx[0][kb + k], w.kbx[1][kb + k], w.kbx[2][kb + k], w.kbx[3][kb + k], w.kbx[4][kb + k], jx1, jy1, jx2, jy2, ja, iou_thr)) {
              sup[ci] = 1;
              break;
            }
          }
        }
        // the block's own bit matrix: row r, columns [4 * q, 4 * q + 4)
        const int r = tid / 16, q = tid % 16;
        if (r < ns) {
          unsigned long long bits = 0ull;
          for (int jj = 4 * q; jj < 4 * q + 4; ++jj)
            if (jj > r && jj < ns &&
                sgb_nms::suppresses(cb[0][r], cb[1][r], cb[2][r], cb[3][r], cb[4][r], cb[0][jj], cb[1][jj], cb[2][jj], cb[3][jj], cb[4][jj], iou_thr))
              bits |= 1ull << jj;
          if (bits) atomicOr(&mask[r], bits);
        }
      }
      __syncthreads();
      if (tid == 0) {
        unsigned long long remv = 0ull, kmask = 0ull;
        for (int r = 0; r < ns; ++r) {
          if (sup[r] || ((remv >> r) & 1ull)) continue;
          kmask |= 1ull << r;
          remv |= mask[r];
        }
        s_kmask = kmask;
      }
      __syncthreads();
      const unsigned long long kmask = s_kmask;
      if (tid < ns && ((kmask >> tid) & 1ull)) {
        const int64_t p = kb + nk + __popcll(kmask & ((1ull << tid) - 1ull));
        for (int f = 0; f < 5; ++f) w.kbx[f][p] = cb[f][tid];
        w.keep[o + cidx[s0 + tid]] = 1;
      }
      nk += __popcll(kmask);
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(NT, 1) sw_merge_output_kernel(int cap, int np2, MergeWs w, float* __restrict__ out, int* __restrict__ out_count) {
  __shared__ int warp_sums[32];
  __shared__ int s_total;
  const int b = blockIdx.x, tid = threadIdx.x;
  const ImageMeta mt = w.meta[b];
  const int64_t o = (int64_t)b * cap;
  if (mt.status != 0) {  // refused: the count is the negated status
    if (tid == 0) out_count[b] = -mt.status;
    return;
  }
  int nout = 0;
  for (int base = 0; base < mt.n; base += NT) {
    const int i = base + tid;
    const bool k = i < mt.n && w.keep[o + i];
    const int pos = block_exclusive_scan(k ? 1 : 0, warp_sums, &s_total);
    if (k) {
      const int p = (int)(w.keys[(int64_t)b * np2 + i] & 0xffffffffu);
      float* r = out + (o + nout + pos) * 6;
      r[0] = w.ox[0][o + p];
      r[1] = w.ox[1][o + p];
      r[2] = w.ox[2][o + p];
      r[3] = w.ox[3][o + p];
      r[4] = w.score[o + p];
      r[5] = (float)w.label[o + p];
    }
    nout += s_total;
  }
  if (tid == 0) out_count[b] = nout;
}

}  // namespace

static int64_t align256(int64_t v) { return (v + 255) / 256 * 256; }

// capacity (rows) of one image and the per-image length of the sort network; -1 when the tile table is malformed
static int merge_dims(int32_t B, const int32_t* image_tiles_host, int32_t T, int32_t P, int64_t* cap, int64_t* np2) {
  if (B <= 0 || T < 0 || P <= 0 || !image_tiles_host || image_tiles_host[0] != 0 || image_tiles_host[B] != T) return -1;
  int64_t mx = 0;
  for (int b = 0; b < B; ++b) {
    const int64_t nt = (int64_t)image_tiles_host[b + 1] - image_tiles_host[b];
    if (nt < 0) return -1;
    mx = nt > mx ? nt : mx;
  }
  *cap = mx * P;
  int64_t p2 = SORT_TILE;
  while (p2 < *cap) p2 <<= 1;
  *np2 = p2;
  return 0;
}

static int64_t merge_bytes(int32_t B, int64_t cap, int64_t np2, int32_t ncls) {
  const int64_t slot = align256((int64_t)B * cap * 4);
  return 18 * slot + align256((int64_t)B * np2 * 8) + align256((int64_t)B * (ncls + 1) * 4) + align256((int64_t)B * sizeof(ImageMeta));
}

extern "C" int64_t sgb_sliding_window_merge_workspace_bytes(int32_t B, const int32_t* image_tiles_host, int32_t T, int32_t P, int32_t ncls) {
  int64_t cap, np2;
  if (merge_dims(B, image_tiles_host, T, P, &cap, &np2) != 0 || ncls <= 0) return 0;
  return merge_bytes(B, cap, np2, ncls);
}

extern "C" int sgb_sliding_window_gather(const sgb_bf16* canvas, int32_t B, int32_t H, int32_t W, int32_t pitch, const int32_t* tiles_host,
                                         const int32_t* tiles, int32_t T, int32_t tile, sgb_bf16* out, void* stream) {
  SGB_REQUIRE(canvas && tiles_host && tiles && out, "null pointer");
  SGB_REQUIRE(B > 0 && H > 0 && W > 0 && tile > 0 && T > 0, "bad dims");
  SGB_REQUIRE(pitch > 0 && pitch % 8 == 0, "channel pitch must be a positive multiple of 8 (16-byte pixels)");
  SGB_REQUIRE(((uintptr_t)canvas & 15) == 0 && ((uintptr_t)out & 15) == 0, "canvas and output must be 16-byte aligned");
  for (int t = 0; t < T; ++t)
    SGB_REQUIRE(tiles_host[3 * t] >= 0 && tiles_host[3 * t] < B && tiles_host[3 * t + 1] >= 0 && tiles_host[3 * t + 2] >= 0,
                "tile table: image index out of range or negative origin");
  const int vec = pitch / 8;
  const int64_t total = (int64_t)T * tile * tile * vec;
  const int grid = (int)((total + 255) / 256 > 132 * 16 ? 132 * 16 : (total + 255) / 256);
  sw_gather_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const uint4*>(canvas), B, H, W, vec, tiles, T, tile,
                                                           reinterpret_cast<uint4*>(out));
  SGB_LAUNCH_CHECK("sw_gather_kernel");
  return SGB_OK;
}

extern "C" int sgb_sliding_window_merge(const float* rows, const int32_t* counts, const int32_t* tiles, const int32_t* image_tiles_host,
                                        const int32_t* image_tiles, int32_t B, int32_t T, int32_t P, int32_t ncls, double iou_thr, float* out,
                                        int32_t* out_count, void* workspace, int64_t workspace_bytes, void* stream) {
  SGB_REQUIRE(rows && counts && tiles && image_tiles_host && image_tiles && out && out_count && workspace, "null pointer");
  SGB_REQUIRE(ncls > 0 && ncls <= MAX_CLASSES, "ncls must be in [1, 4096]");
  int64_t cap, np2;
  SGB_REQUIRE(merge_dims(B, image_tiles_host, T, P, &cap, &np2) == 0, "image_tiles must be ascending from 0 to T");
  SGB_REQUIRE(T > 0, "no tiles");
  SGB_REQUIRE(np2 <= (1ll << 30), "more than 2^30 candidate rows for one image");
  SGB_REQUIRE(workspace_bytes >= merge_bytes(B, cap, np2, ncls), "workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* p = reinterpret_cast<unsigned char*>(workspace);
  const int64_t slot = align256((int64_t)B * cap * 4);
  MergeWs w;
  auto f = [&]() {
    float* r = reinterpret_cast<float*>(p);
    p += slot;
    return r;
  };
  for (int i = 0; i < 4; ++i) w.ox[i] = f();
  w.score = f();
  w.label = reinterpret_cast<int*>(f());
  for (int i = 0; i < 4; ++i) w.sbx[i] = f();
  w.sarea = f();
  w.slabel = reinterpret_cast<int*>(f());
  w.keep = reinterpret_cast<int*>(f());
  for (int i = 0; i < 5; ++i) w.kbx[i] = f();
  w.keys = reinterpret_cast<unsigned long long*>(p);
  p += align256((int64_t)B * np2 * 8);
  w.cls_off = reinterpret_cast<int*>(p);
  p += align256((int64_t)B * (ncls + 1) * 4);
  w.meta = reinterpret_cast<ImageMeta*>(p);
  const int icap = (int)cap, inp2 = (int)np2;

  sw_compact_kernel<<<B, NT, 0, st>>>(rows, counts, tiles, image_tiles, P, ncls, icap, inp2, w);
  SGB_LAUNCH_CHECK("sw_compact_kernel");
  const dim3 tiles_grid(inp2 / SORT_TILE, B);
  sw_sort_local_kernel<<<tiles_grid, NT, 0, st>>>(w.keys, inp2, 2, SORT_TILE);
  SGB_LAUNCH_CHECK("sw_sort_local_kernel");
  for (int k = 2 * SORT_TILE; k <= inp2; k <<= 1) {
    for (int j = k >> 1; j >= SORT_TILE; j >>= 1) {
      sw_sort_global_kernel<<<dim3((inp2 / 2 + 255) / 256, B), 256, 0, st>>>(w.keys, inp2, k, j);
      SGB_LAUNCH_CHECK("sw_sort_global_kernel");
    }
    sw_sort_local_kernel<<<tiles_grid, NT, 0, st>>>(w.keys, inp2, k, k);
    SGB_LAUNCH_CHECK("sw_sort_local_kernel (merge)");
  }
  const int gx = (int)((cap + 255) / 256 > 64 ? 64 : (cap + 255) / 256);
  sw_gather_sorted_kernel<<<dim3(gx, B), 256, 0, st>>>(icap, inp2, w);
  SGB_LAUNCH_CHECK("sw_gather_sorted_kernel");
  sw_merge_nms_kernel<<<dim3(ncls, B), NT, 0, st>>>(icap, ncls, iou_thr, w);
  SGB_LAUNCH_CHECK("sw_merge_nms_kernel");
  sw_merge_output_kernel<<<B, NT, 0, st>>>(icap, inp2, w, out, out_count);
  SGB_LAUNCH_CHECK("sw_merge_output_kernel");
  return SGB_OK;
}

// kernels launched by sgb_sliding_window_merge for the given dimensions (the Python launch counter)
extern "C" int32_t sgb_sliding_window_merge_launches(int32_t B, const int32_t* image_tiles_host, int32_t T, int32_t P) {
  int64_t cap, np2;
  if (merge_dims(B, image_tiles_host, T, P, &cap, &np2) != 0) return 0;
  int n = 5;
  for (int64_t k = 2 * SORT_TILE; k <= np2; k <<= 1) {
    for (int64_t j = k >> 1; j >= SORT_TILE; j >>= 1) ++n;
    ++n;
  }
  return n;
}
