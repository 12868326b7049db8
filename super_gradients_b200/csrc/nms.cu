// Batched, class-aware NMS: one CTA (1024 threads) per image does
//   threshold -> (radix-select top-k if needed) -> ordered compaction -> bitonic sort -> IoU bit-matrix -> greedy sweep
// entirely in shared memory, reproducing index-for-index what the reference does per image in Python:
//   PPYoloEPostPredictionCallback.forward  (training/models/detection_models/pp_yolo_e/post_prediction_callback.py:42-98)
//   YoloNASPosePostPredictionCallback      (…/yolo_nas_pose/yolo_nas_pose_post_prediction_callback.py:38-94)
//   torchvision.ops.boxes.batched_nms / nms (torchvision 0.26: ops/boxes.py:43-120 and csrc/ops/cpu/nms_kernel.cpp)
//
// Bit-exactness notes (all mirrored here):
//   * candidates are enumerated row-major (anchor, class), `score > thr` in fp32 (multi-label) or `>=` (single-label);
//   * if there are more than top_k candidates, torch.topk(sorted) picks them (ties: we take the lowest index);
//   * torchvision sorts by score with a STABLE descending sort, so ties keep candidate-list order;
//   * batched_nms uses the coordinate trick when 4*n <= 4000 on CPU, otherwise per-class NMS on the raw boxes;
//   * IoU arithmetic is fp32 with no fused multiply-add, and `ovr > iou_threshold` is evaluated in double.
#include "common.cuh"
#include "nms_math.cuh"

#include <math.h>

namespace {

constexpr int NT = 1024;      // threads per CTA
constexpr int KMAX = 1024;    // max candidates entering NMS
constexpr int NBIN = 2048;

struct NmsSmem {
  unsigned long long mask[KMAX * (KMAX / 64)];  // 128 KB
  unsigned long long keys[KMAX];                // sort keys
  int flat[KMAX];                               // candidate flat index by candidate position
  float bx[4][KMAX];                            // (offset) boxes in sorted order
  float area[KMAX];
  int label[KMAX];
  int sflat[KMAX];                              // flat index in sorted order
  int hist[NBIN];
  int wcnt[32], wtie[32];
  int kept[KMAX];
  int misc[16];
  float fmisc[4];
};

__device__ __forceinline__ unsigned okey(float f) { return sgb_nms::score_key(f); }

__device__ __forceinline__ bool passes(float s, float thr, int incl) { return incl ? (s >= thr) : (s > thr); }

// argmax pre-pass for single-label mode (torch.max(dim=1): first maximal index, or the first NaN and its index -- a NaN maximum
// then fails the threshold and drops the anchor)
__global__ void nms_argmax_kernel(const float* __restrict__ scores, int64_t rows, int C, float* conf, int* lab) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < rows; i += (int64_t)gridDim.x * blockDim.x) {
    float best = scores[i * C];
    int bi = 0;
    for (int c = 1; c < C && best == best; ++c) {
      float v = scores[i * C + c];
      if (v > best || v != v) {
        best = v;
        bi = c;
      }
    }
    conf[i] = best;
    lab[i] = bi;
  }
}

// histogram of `shift`-ed key digits over this warp's segment, restricted to keys whose higher bits equal `prefix`
template <int BITS>
__device__ void hist_pass(const float* __restrict__ sc, int seg0, int seg1, float thr, int incl, unsigned prefix_mask,
                          unsigned prefix, int shift, int* hist, int lane) {
  for (int base = seg0; base < seg1; base += 128) {
    float v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      int idx = base + u * 32 + lane;
      v[u] = idx < seg1 ? sc[idx] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      int idx = base + u * 32 + lane;
      if (idx < seg1 && passes(v[u], thr, incl)) {
        unsigned k = okey(v[u]);
        // (warp-aggregating equal bins with __match_any_sync was measured slower here: 211 vs 179 us for the pre-filter launch)
        if ((k & prefix_mask) == prefix) atomicAdd(&hist[(k >> shift) & ((1u << BITS) - 1)], 1);
      }
    }
  }
}

// warp 0: find the bin holding the `need`-th largest element; returns bin, writes remaining need
__device__ int find_bin(const int* hist, int nbins, int need, int lane, int* need_out) {
  const int per = nbins / 32;
  int s = 0;
  for (int j = 0; j < per; ++j) s += hist[lane * per + j];
  // suffix sum over lanes (lane 31 holds the largest keys)
  int suf = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_down_sync(0xffffffffu, suf, o);
    if (lane + o < 32) suf += t;
  }
  int above = suf - s;  // elements in lanes above mine
  bool mine = above < need && suf >= need;
  unsigned ball = __ballot_sync(0xffffffffu, mine);
  int owner = 31 - __clz(ball);  // exactly one lane satisfies it when total >= need
  int bin = 0, rem = 0;
  if (lane == owner) {
    int cum = above;
    for (int j = per - 1; j >= 0; --j) {
      int h = hist[lane * per + j];
      if (cum + h >= need) {
        bin = lane * per + j;
        rem = need - cum;
        break;
      }
      cum += h;
    }
  }
  bin = __shfl_sync(0xffffffffu, bin, owner);
  rem = __shfl_sync(0xffffffffu, rem, owner);
  *need_out = rem;
  return bin;
}

// Scratch of the selection phase (shared memory of the calling kernel)
struct SelScratch {
  int* hist;  // [NBIN]
  int* wcnt;  // [32]
  int* wtie;  // [32]
  int* misc;  // [16]
};

// Selection phase shared by the NMS kernel and its pre-filter: among sc[0, n_items) the entries passing the threshold, or -- when
// more than top_k pass -- the top_k largest (3-level radix select; equal scores: lowest index first), visited in INDEX order.
// emit(p, idx, key) is called once per selected entry with its output position p (0 .. nsel-1, increasing with idx).  All NT
// threads of the CTA call it; returns the number selected.  `sc` may point to global or shared memory.
template <class Emit>
__device__ int select_ordered(const float* __restrict__ sc, const int n_items, const float thr, const int incl, const int top_k, const SelScratch sh,
                              Emit&& emit) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  // contiguous segment per warp (multiple of 128 items so that the unrolled loop stays in order)
  int seg_len = (n_items + 31) / 32;
  seg_len = ((seg_len + 127) / 128) * 128;
  const int seg0 = min(warp * seg_len, n_items), seg1 = min(seg0 + seg_len, n_items);

  // ---- pass 1: level-1 histogram (top 11 key bits) + per-warp candidate counts
  for (int i = t; i < NBIN; i += NT) sh.hist[i] = 0;
  __syncthreads();
  hist_pass<11>(sc, seg0, seg1, thr, incl, 0u, 0u, 21, sh.hist, lane);
  __syncthreads();
  if (warp == 0) {
    int s = 0;
    for (int j = 0; j < NBIN / 32; ++j) s += sh.hist[lane * (NBIN / 32) + j];
    int tot = s;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
    if (lane == 0) sh.misc[0] = tot;
  }
  __syncthreads();
  const int total = sh.misc[0];
  unsigned Tkey = 0;  // select keys > Tkey, plus `tie_need` keys == Tkey (lowest index first)
  int tie_need = 0;
  bool select_all = total <= top_k;
  if (!select_all) {
    // 3-level radix select of the top_k-th largest key
    if (warp == 0) {
      int need;
      int b1 = find_bin(sh.hist, NBIN, top_k, lane, &need);
      if (lane == 0) {
        sh.misc[1] = b1;
        sh.misc[2] = need;
      }
    }
    __syncthreads();
    unsigned prefix = (unsigned)sh.misc[1] << 21;
    int need = sh.misc[2];
    for (int i = t; i < NBIN; i += NT) sh.hist[i] = 0;
    __syncthreads();
    hist_pass<11>(sc, seg0, seg1, thr, incl, 0xffe00000u, prefix, 10, sh.hist, lane);
    __syncthreads();
    if (warp == 0) {
      int need2;
      int b2 = find_bin(sh.hist, NBIN, need, lane, &need2);
      if (lane == 0) {
        sh.misc[1] = b2;
        sh.misc[2] = need2;
      }
    }
    __syncthreads();
    prefix |= (unsigned)sh.misc[1] << 10;
    need = sh.misc[2];
    for (int i = t; i < NBIN; i += NT) sh.hist[i] = 0;
    __syncthreads();
    hist_pass<10>(sc, seg0, seg1, thr, incl, 0xfffffc00u, prefix, 0, sh.hist, lane);
    __syncthreads();
    if (warp == 0) {
      int need3;
      int b3 = find_bin(sh.hist, 1024, need, lane, &need3);
      if (lane == 0) {
        sh.misc[1] = b3;
        sh.misc[2] = need3;
      }
    }
    __syncthreads();
    Tkey = prefix | (unsigned)sh.misc[1];
    tie_need = sh.misc[2];
  }

  // ---- count pass: per-warp (# selected strictly above, # ties) in index order
  {
    int cg = 0, ct = 0;
    for (int base = seg0; base < seg1; base += 128) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        int idx = base + u * 32 + lane;
        if (idx < seg1) {
          float v = sc[idx];
          if (passes(v, thr, incl)) {
            unsigned k = okey(v);
            if (select_all || k > Tkey) ++cg;
            else if (k == Tkey) ++ct;
          }
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      cg += __shfl_xor_sync(0xffffffffu, cg, o);
      ct += __shfl_xor_sync(0xffffffffu, ct, o);
    }
    if (lane == 0) {
      sh.wcnt[warp] = cg;
      sh.wtie[warp] = ct;
    }
  }
  __syncthreads();
  if (t == 0) {
    // exclusive scan over warps; ties are granted in index order until tie_need is exhausted
    int pos = 0, ties_before = 0;
    for (int w = 0; w < 32; ++w) {
      int cg = sh.wcnt[w], ct = sh.wtie[w];
      int grant = 0;
      if (!select_all) {
        int left = tie_need - ties_before;
        grant = left > 0 ? (ct < left ? ct : left) : 0;
      }
      sh.wcnt[w] = pos;           // output base of this warp
      sh.wtie[w] = ties_before;   // ties preceding this warp
      pos += cg + grant;
      ties_before += ct;
    }
    sh.misc[3] = pos;  // number of selected candidates
  }
  __syncthreads();
  const int nsel = sh.misc[3];

  // ---- write pass: ordered compaction into S.flat / S.keys
  {
    int pos = sh.wcnt[warp];
    int ties_seen = sh.wtie[warp];
    for (int base = seg0; base < seg1; base += 128) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        int idx = base + u * 32 + lane;
        bool valid = false, tie = false;
        unsigned k = 0;
        if (idx < seg1) {
          float v = sc[idx];
          if (passes(v, thr, incl)) {
            k = okey(v);
            if (select_all || k > Tkey) valid = true;
            else if (k == Tkey) tie = true;
          }
        }
        unsigned tb = __ballot_sync(0xffffffffu, tie);
        if (tie) {
          int rank = ties_seen + __popc(tb & ((1u << lane) - 1));
          if (rank < tie_need) valid = true;
        }
        ties_seen += __popc(tb);
        unsigned vb = __ballot_sync(0xffffffffu, valid);
        if (valid) {
          int p = pos + __popc(vb & ((1u << lane) - 1));
          if (p < top_k) emit(p, idx, k);
        }
        pos += __popc(vb);
      }
    }
  }
  __syncthreads();

  __syncthreads();
  return nsel;
}

// Pre-filter of the multi-label path.  One CTA per (slice, image): the slice of the score row (<= PF_SLICE floats) is read from
// HBM ONCE with 16-byte loads into shared memory; the selection phase then runs on the shared-memory copy and writes the slice's
// candidates -- everything passing the threshold, or the slice's own top_k -- in index order to cand_sc / cand_flat[b][slice][0..top_k),
// padding the segment with -inf.  The union of the per-slice top_k contains the image's top_k (an entry beaten by fewer than
// top_k entries of the image is beaten by fewer than top_k entries of its slice; ties keep the lowest index in both rules), and the
// concatenated segments keep the row-major candidate order, so nms_kernel run on the candidate lists selects, orders and suppresses
// exactly what it would on the full row.  The full row is L * ncls floats per image (2.7 MB for 8400 x 80): scanned by one CTA per
// image with up to five passes of 4-byte loads it was the whole cost of the launch (1.77 ms for 32 images: 51 GB/s); here every SM
// streams slices.
constexpr int PF_SLICE = 24576;  // floats per slice: 96 KB + scratch, two CTAs per SM
__global__ void __launch_bounds__(NT, 2) nms_prefilter_kernel(SgbNmsDesc d, const float* __restrict__ scores, int n_items, int slice_len, int nslices,
                                                              float* __restrict__ cand_sc, int* __restrict__ cand_flat) {
  extern __shared__ __align__(16) unsigned char pf_raw[];
  float* v = reinterpret_cast<float*>(pf_raw);             // [slice_len]
  int* scratch = reinterpret_cast<int*>(v + PF_SLICE);      // hist[NBIN], wcnt[32], wtie[32], misc[16]
  const int s = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
  const int i0 = s * slice_len;
  const int n = max(0, min(slice_len, n_items - i0));
  const float* src = scores + (int64_t)b * n_items + i0;
  if (((uintptr_t)src & 15) == 0) {
    const int n4 = n >> 2;
    for (int i = t; i < n4; i += NT) reinterpret_cast<float4*>(v)[i] = __ldg(reinterpret_cast<const float4*>(src) + i);
    for (int i = (n4 << 2) + t; i < n; i += NT) v[i] = src[i];
  } else {
    for (int i = t; i < n; i += NT) v[i] = src[i];
  }
  __syncthreads();
  const int top_k = d.top_k < KMAX ? d.top_k : KMAX;
  float* osc = cand_sc + ((int64_t)b * nslices + s) * top_k;
  int* ofl = cand_flat + ((int64_t)b * nslices + s) * top_k;
  SelScratch sh{scratch, scratch + NBIN, scratch + NBIN + 32, scratch + NBIN + 64};
  const int nsel = select_ordered(v, n, d.score_thr, d.thr_inclusive, top_k, sh, [&](int p, int idx, unsigned) {
    osc[p] = v[idx];
    ofl[p] = i0 + idx;
  });
  for (int j = nsel + t; j < top_k; j += NT) {
    osc[j] = -INFINITY;  // never passes a (finite) threshold
    ofl[j] = 0;
  }
}

// Split form of the per-image work for large candidate counts.  With ~1000 candidates the IoU bit-matrix is 500 k IoU evaluations
// (fp32 division each) and dominated the one-CTA-per-image kernel (32 CTAs on 132 SMs); it is the only part with no sequential
// dependence, so it runs as its own launch over (row block, image) CTAs between a "front" launch (selection, sort, gather, offsets,
// areas -> NmsStage in global memory) and a "back" launch (greedy sweep over the matrix + output rows).  Same arithmetic, same
// order of operations per IoU.
struct NmsStage {
  float bx[4][KMAX];
  float area[KMAX];
  int label[KMAX];
  int sflat[KMAX];
  int nsel, trick, pad_[2];
};
constexpr int MASK_ROWS = 64;  // rows of the bit-matrix per CTA of nms_mask_kernel

__global__ void __launch_bounds__(NT, 1) nms_mask_kernel(SgbNmsDesc d, const NmsStage* __restrict__ stages, unsigned long long* __restrict__ masks) {
  __shared__ float bx[4][KMAX];
  __shared__ float area[KMAX];
  __shared__ int label[KMAX];
  const int b = blockIdx.y, t = threadIdx.x;
  const NmsStage& st = stages[b];
  const int nsel = st.nsel;
  const int i0 = blockIdx.x * MASK_ROWS;
  if (i0 >= nsel) return;
  for (int i = t; i < nsel; i += NT) {
    bx[0][i] = st.bx[0][i];
    bx[1][i] = st.bx[1][i];
    bx[2][i] = st.bx[2][i];
    bx[3][i] = st.bx[3][i];
    area[i] = st.area[i];
    label[i] = st.label[i];
  }
  __syncthreads();
  const int nw = (nsel + 63) / 64;
  const bool same_class_only = !d.class_agnostic && !st.trick;
  unsigned long long* mrow = masks + (int64_t)b * KMAX * (KMAX / 64);
  const int rows = min(MASK_ROWS, nsel - i0);
  for (int pair = t; pair < rows * nw; pair += NT) {
    const int w = pair / rows, i = i0 + pair % rows;  // consecutive lanes: consecutive rows of ONE word -> box j is a broadcast read
    unsigned long long bits = 0ull;
    if (w * 64 + 63 > i) {
      const float ix1 = bx[0][i], iy1 = bx[1][i], ix2 = bx[2][i], iy2 = bx[3][i], ia = area[i];
      const int li = label[i];
      const int j0 = w * 64;
      const int jend = min(j0 + 64, nsel);
      for (int j = max(j0, i + 1); j < jend; ++j) {
        if (same_class_only && label[j] != li) continue;
        if (sgb_nms::suppresses(ix1, iy1, ix2, iy2, ia, bx[0][j], bx[1][j], bx[2][j], bx[3][j], area[j], d.iou_thr)) bits |= 1ull << (j - j0);
      }
    }
    mrow[i * (KMAX / 64) + w] = bits;
  }
}

// cand_sc / cand_flat (optional): per image `cand_items` pre-filtered candidates in row-major order (nms_prefilter_kernel); the
// selection phase then scans those instead of the full score row.
__global__ void __launch_bounds__(NT, 1) nms_kernel(SgbNmsDesc d, const float* __restrict__ boxes,
                                                    const float* __restrict__ scores, const float* __restrict__ conf,
                                                    const int* __restrict__ lab, float* out, int* out_idx,
                                                    int* out_count, const float* __restrict__ cand_sc, const int* __restrict__ cand_flat,
                                                    int cand_items, int mode, NmsStage* __restrict__ stages,
                                                    const unsigned long long* __restrict__ masks) {
  // mode 0: everything in this launch; 1: front (up to the areas, staged to `stages`); 2: back (sweep over `masks` + output)
  extern __shared__ __align__(16) unsigned char smem_raw[];
  NmsSmem& S = *reinterpret_cast<NmsSmem*>(smem_raw);
  const int b = blockIdx.x;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const bool multi = d.multi_label != 0;
  const int n_items = multi ? d.L * d.ncls : d.L;
  const float* orig = multi ? scores + (int64_t)b * n_items : conf + (int64_t)b * d.L;  // score of a flat candidate index
  const float* sc = cand_sc ? cand_sc + (int64_t)b * cand_items : orig;
  const int n_scan = cand_sc ? cand_items : n_items;
  const float thr = d.score_thr;
  const int incl = d.thr_inclusive;
  SelScratch sh{S.hist, S.wcnt, S.wtie, S.misc};
  const int top_k = d.top_k < KMAX ? d.top_k : KMAX;
  const int* fmap = cand_flat ? cand_flat + (int64_t)b * cand_items : nullptr;
  if (mode == 2) {  // back half: restore what the sweep and the output rows need
    const NmsStage& st = stages[b];
    const int ns = st.nsel;
    for (int i = t; i < ns; i += NT) {
      S.label[i] = st.label[i];
      S.sflat[i] = st.sflat[i];
    }
    const int nwb = (ns + 63) / 64;
    const unsigned long long* mrow = masks + (int64_t)b * KMAX * (KMAX / 64);
    for (int i = t; i < ns * nwb; i += NT) {
      const int r = i / nwb, w = i - r * nwb;
      S.mask[r * (KMAX / 64) + w] = mrow[r * (KMAX / 64) + w];
    }
    if (t == 0) S.misc[5] = ns;
    __syncthreads();
  }
  const int nsel = mode == 2 ? S.misc[5] : select_ordered(sc, n_scan, thr, incl, top_k, sh, [&](int p, int idx, unsigned k) {
    S.flat[p] = fmap ? fmap[idx] : idx;
    S.keys[p] = ((unsigned long long)(~k) << 32) | (unsigned)p;
  });

  bool trick_flag = false;
  if (mode != 2) {
  // ---- bitonic sort of (score desc, position asc)
  int np2 = 1;
  while (np2 < nsel) np2 <<= 1;
  for (int i = nsel + t; i < np2; i += NT) S.keys[i] = ~0ull;
  __syncthreads();
  for (int k = 2; k <= np2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = t; i < np2; i += NT) {
        int ixj = i ^ j;
        if (ixj > i) {
          unsigned long long a = S.keys[i], c = S.keys[ixj];
          bool up = (i & k) == 0;
          if ((a > c) == up) {
            S.keys[i] = c;
            S.keys[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  }

  // ---- gather boxes / labels in sorted order
  float lmax = -INFINITY;
  for (int i = t; i < nsel; i += NT) {
    int p = (int)(S.keys[i] & 0xffffffffu);
    int f = S.flat[p];
    int anchor = multi ? f / d.ncls : f;
    int label = multi ? f - anchor * d.ncls : (lab ? lab[(int64_t)b * d.L + f] : 0);
    const float* bp = boxes + ((int64_t)b * d.L + anchor) * 4;
    float x1 = bp[0], y1 = bp[1], x2 = bp[2], y2 = bp[3];
    S.bx[0][i] = x1;
    S.bx[1][i] = y1;
    S.bx[2][i] = x2;
    S.bx[3][i] = y2;
    S.label[i] = label;
    S.sflat[i] = f;
    lmax = sgb_nms::max_nan(lmax, sgb_nms::max_nan(sgb_nms::max_nan(x1, y1), sgb_nms::max_nan(x2, y2)));
  }
  // batched_nms path selection exactly as torchvision (CPU): coordinate trick iff boxes.numel() <= 4000
  const bool trick = !d.class_agnostic && (4 * nsel <= 4000);
  trick_flag = trick;
  if (trick) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lmax = sgb_nms::max_nan(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
    float* wmax = reinterpret_cast<float*>(S.hist);
    if (lane == 0) wmax[warp] = lmax;
    __syncthreads();
    if (t == 0) {
      float m = -INFINITY;
      for (int w = 0; w < 32; ++w) m = sgb_nms::max_nan(m, wmax[w]);
      S.fmisc[1] = sgb_nms::offset_step(m);  // max_coordinate + 1
    }
    __syncthreads();
    const float step = S.fmisc[1];
    for (int i = t; i < nsel; i += NT) {
      float off = sgb_nms::label_offset(S.label[i], step);
      S.bx[0][i] = __fadd_rn(S.bx[0][i], off);
      S.bx[1][i] = __fadd_rn(S.bx[1][i], off);
      S.bx[2][i] = __fadd_rn(S.bx[2][i], off);
      S.bx[3][i] = __fadd_rn(S.bx[3][i], off);
    }
  }
  __syncthreads();
  for (int i = t; i < nsel; i += NT)
    S.area[i] = sgb_nms::area(S.bx[0][i], S.bx[1][i], S.bx[2][i], S.bx[3][i]);
  __syncthreads();

  }
  if (mode == 1) {  // front half done: stage what the matrix and the back half need
    NmsStage& st = stages[b];
    for (int i = t; i < nsel; i += NT) {
      st.bx[0][i] = S.bx[0][i];
      st.bx[1][i] = S.bx[1][i];
      st.bx[2][i] = S.bx[2][i];
      st.bx[3][i] = S.bx[3][i];
      st.area[i] = S.area[i];
      st.label[i] = S.label[i];
      st.sflat[i] = S.sflat[i];
    }
    if (t == 0) {
      st.nsel = nsel;
      st.trick = trick_flag ? 1 : 0;
    }
    return;
  }
  const int nw = (nsel + 63) / 64;
  if (mode == 0) {
  // ---- IoU bit matrix: mask[i][w] bit j: j > i, suppressed by i
  const bool same_class_only = !d.class_agnostic && !trick_flag;
  for (int pair = t; pair < nsel * nw; pair += NT) {
    int w = pair / nsel, i = pair - w * nsel;  // consecutive lanes: consecutive rows of ONE word -> box j is a broadcast read
    unsigned long long bits = 0ull;
    if (w * 64 + 63 > i) {
      float ix1 = S.bx[0][i], iy1 = S.bx[1][i], ix2 = S.bx[2][i], iy2 = S.bx[3][i], ia = S.area[i];
      int li = S.label[i];
      int j0 = w * 64;
      int jend = min(j0 + 64, nsel);
      for (int j = max(j0, i + 1); j < jend; ++j) {
        if (same_class_only && S.label[j] != li) continue;
        if (sgb_nms::suppresses(ix1, iy1, ix2, iy2, ia, S.bx[0][j], S.bx[1][j], S.bx[2][j], S.bx[3][j], S.area[j], d.iou_thr)) bits |= 1ull << (j - j0);
      }
    }
    S.mask[i * (KMAX / 64) + w] = bits;
  }
  __syncthreads();

  }
  // ---- greedy sweep by warp 0: lane w owns word w of the "removed" bitset
  if (warp == 0) {
    unsigned long long remv = 0ull;  // lanes 0..15
    int nkeep = 0;
    for (int i = 0; i < nsel; ++i) {
      unsigned long long wv = __shfl_sync(0xffffffffu, remv, i >> 6);
      if (!((wv >> (i & 63)) & 1ull)) {
        if (lane == 0) S.kept[nkeep] = i;
        ++nkeep;
        if (nkeep >= d.max_out) break;
        if (lane < nw) remv |= S.mask[i * (KMAX / 64) + lane];
      }
    }
    if (lane == 0) S.misc[4] = nkeep;
  }
  __syncthreads();
  const int nkeep = S.misc[4];
  if (t == 0) out_count[b] = nkeep;
  for (int r = t; r < d.max_out; r += NT) {
    float* o = out + ((int64_t)b * d.max_out + r) * 6;
    if (r < nkeep) {
      int i = S.kept[r];
      int f = S.sflat[i];
      int anchor = multi ? f / d.ncls : f;
      const float* bp = boxes + ((int64_t)b * d.L + anchor) * 4;
      o[0] = bp[0];
      o[1] = bp[1];
      o[2] = bp[2];
      o[3] = bp[3];
      o[4] = orig[f];
      o[5] = (float)S.label[i];
      out_idx[(int64_t)b * d.max_out + r] = multi ? f : f * d.ncls + S.label[i];
    } else {
      o[0] = o[1] = o[2] = o[3] = o[4] = o[5] = 0.f;
      out_idx[(int64_t)b * d.max_out + r] = -1;
    }
  }
}

}  // namespace

// multi-label rows longer than this go through the pre-filter
static bool prefilter_wanted(const SgbNmsDesc* d) {
  return d->multi_label && (int64_t)d->L * d->ncls > 4 * PF_SLICE && (int64_t)d->L * d->ncls < (1ll << 30) && isfinite(d->score_thr);
}
static int prefilter_slices(const SgbNmsDesc* d, int* slice_len) {
  const int64_t n = (int64_t)d->L * d->ncls;
  const int ns = (int)((n + PF_SLICE - 1) / PF_SLICE);
  int sl = (int)((n + ns - 1) / ns);
  sl = ((sl + 3) / 4) * 4;  // slice starts stay 16-byte aligned when the row is
  *slice_len = sl;
  return (int)((n + sl - 1) / sl);
}

// more than this many candidates per image: front / IoU-matrix / back as three launches
static bool split_wanted(const SgbNmsDesc* d) {
  return d->top_k > 512;
}
static int64_t align256(int64_t v) { return (v + 255) / 256 * 256; }
// workspace layout: [single-label conf / labels  |  pre-filter candidates] [stages] [masks]
static int64_t ws_head_bytes(const SgbNmsDesc* d) {
  int64_t bytes = (int64_t)d->B * d->L * 8;
  if (prefilter_wanted(d)) {
    int sl;
    const int ns = prefilter_slices(d, &sl);
    const int64_t cand = (int64_t)d->B * ns * (d->top_k < KMAX ? d->top_k : KMAX) * 8;
    if (cand > bytes) bytes = cand;
  }
  return align256(bytes);
}

extern "C" int64_t sgb_nms_workspace_bytes(const SgbNmsDesc* d) {
  if (!d) return 0;
  int64_t bytes = ws_head_bytes(d) + 256;
  if (split_wanted(d)) bytes += align256((int64_t)d->B * sizeof(NmsStage)) + (int64_t)d->B * KMAX * (KMAX / 64) * 8;
  return bytes;
}

extern "C" int sgb_batched_nms(const SgbNmsDesc* d, const float* boxes, const float* scores, float* out,
                               int32_t* out_idx, int32_t* out_count, void* workspace, int64_t workspace_bytes,
                               void* stream) {
  SGB_REQUIRE(d && boxes && scores && out && out_idx && out_count, "null pointer");
  SGB_REQUIRE(d->B > 0 && d->L > 0 && d->ncls > 0, "bad dims");
  SGB_REQUIRE(d->max_out > 0 && d->max_out <= KMAX, "max_out must be in [1, 1024]");
  SGB_REQUIRE(d->top_k > 0, "top_k must be positive");
  if (d->top_k > KMAX) {
    sgb_set_error("sgb_batched_nms: top_k %d > %d is not supported by the shared-memory IoU matrix", d->top_k, KMAX);
    return SGB_E_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* conf = nullptr;
  int* lab = nullptr;
  if (!d->multi_label) {
    SGB_REQUIRE(workspace && workspace_bytes >= sgb_nms_workspace_bytes(d), "workspace too small");
    conf = reinterpret_cast<float*>(workspace);
    lab = reinterpret_cast<int*>(conf + (int64_t)d->B * d->L);
    int64_t rows = (int64_t)d->B * d->L;
    int grid = (int)((rows + 255) / 256 > 132 * 8 ? 132 * 8 : (rows + 255) / 256);
    nms_argmax_kernel<<<grid, 256, 0, st>>>(scores, rows, d->ncls, conf, lab);
    SGB_LAUNCH_CHECK("nms_argmax_kernel");
  }
  static bool attr = false;
  if (!attr) {
    if (int rc = sgb_cuda_check(
            cudaFuncSetAttribute(nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(NmsSmem)),
            "cudaFuncSetAttribute(nms_kernel)"))
      return rc;
    attr = true;
  }
  const float* cand_sc = nullptr;
  const int* cand_flat = nullptr;
  int cand_items = 0;
  if (prefilter_wanted(d) && workspace && workspace_bytes >= sgb_nms_workspace_bytes(d)) {
    int sl;
    const int ns = prefilter_slices(d, &sl);
    const int tk = d->top_k < KMAX ? d->top_k : KMAX;
    float* csc = reinterpret_cast<float*>(workspace);
    int* cfl = reinterpret_cast<int*>(csc + (int64_t)d->B * ns * tk);
    const size_t pf_smem = (size_t)PF_SLICE * 4 + (NBIN + 32 + 32 + 16) * 4;
    static bool pf_attr = false;
    if (!pf_attr) {
      if (int rc = sgb_cuda_check(cudaFuncSetAttribute(nms_prefilter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pf_smem),
                                  "cudaFuncSetAttribute(nms_prefilter_kernel)"))
        return rc;
      pf_attr = true;
    }
    nms_prefilter_kernel<<<dim3(ns, d->B), NT, pf_smem, st>>>(*d, scores, d->L * d->ncls, sl, ns, csc, cfl);
    SGB_LAUNCH_CHECK("nms_prefilter_kernel");
    cand_sc = csc;
    cand_flat = cfl;
    cand_items = ns * tk;
  }
  if (split_wanted(d) && workspace && workspace_bytes >= sgb_nms_workspace_bytes(d)) {
    unsigned char* base = reinterpret_cast<unsigned char*>(workspace) + ws_head_bytes(d);
    NmsStage* stages = reinterpret_cast<NmsStage*>(base);
    unsigned long long* masks = reinterpret_cast<unsigned long long*>(base + align256((int64_t)d->B * sizeof(NmsStage)));
    nms_kernel<<<d->B, NT, sizeof(NmsSmem), st>>>(*d, boxes, scores, conf, lab, out, out_idx, out_count, cand_sc, cand_flat, cand_items, 1, stages, masks);
    SGB_LAUNCH_CHECK("nms_kernel (front)");
    nms_mask_kernel<<<dim3(KMAX / MASK_ROWS, d->B), NT, 0, st>>>(*d, stages, masks);
    SGB_LAUNCH_CHECK("nms_mask_kernel");
    nms_kernel<<<d->B, NT, sizeof(NmsSmem), st>>>(*d, boxes, scores, conf, lab, out, out_idx, out_count, cand_sc, cand_flat, cand_items, 2, stages, masks);
    SGB_LAUNCH_CHECK("nms_kernel (back)");
    return SGB_OK;
  }
  nms_kernel<<<d->B, NT, sizeof(NmsSmem), st>>>(*d, boxes, scores, conf, lab, out, out_idx, out_count, cand_sc, cand_flat, cand_items, 0, nullptr, nullptr);
  SGB_LAUNCH_CHECK("nms_kernel");
  return SGB_OK;
}
