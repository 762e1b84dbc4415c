// label_rle.cu — a semantic label map as one COCO run-length code per label, without a mask per label.
//
// detectron2's SemSegEvaluator.process (encode_json_sem_seg) runs np.unique over the predicted label map, builds the boolean
// mask of every label present and hands each to mask_util.encode: one full pass over the image per label, on the host.  The
// code of label c only depends on where c starts and stops in column-major order t = x * H + y: c changes state exactly at the
// boundaries t >= 1 with L(t) != L(t - 1) where c is one of the two labels, and at t = 0 when L(0) = c (a leading run of 0
// zeros).  Its counts are the differences of [0, those positions..., H * W].  Passes:
//
//   lrle_columns_kernel    one warp per column: boundaries per column, a bitmap of the labels present
//   lrle_compact_kernel    the present labels in ascending order (P of them), their number of boundaries m, and whether the
//                          codes can fit the output at all (every count takes at least one character)
//   lrle_count_kernel      events per (present label, column) -> [P, W] int32, then an exclusive scan in label-major order
//   lrle_positions_kernel  one warp per column: each event's position, written in order at its (label, column) offset; the
//                          rank of an event among the warp's 32 pixels comes from __match_any_sync masks, no atomics
//   lrle_chars_kernel      per count: its rleToString length (LEN) or its characters (at the scanned offsets)
//
// Every value is a count or a scanned sum of counts, so the output does not depend on the order of the atomics in the count
// pass.  Output (a "codes" body): P x (int32 label, int32 character offset, int32 character length), then the characters.
// The packed variant (ape_label_rle_pack) writes one image's semantic slot and falls back to the map as uint16 when the codes
// do not fit.
#include <algorithm>

#include "common.cuh"
#include "rle.cuh"

namespace ape {
namespace {

constexpr int LRLE_LABELS = 65536, LRLE_WORDS = LRLE_LABELS / 32;
constexpr int LRLE_ITEMS = 8, LRLE_TILE = 256 * LRLE_ITEMS;  // scan tile: 8 ints per thread
constexpr unsigned FULL = 0xffffffffu;
// words of the state block: slot kind and bytes, P, m, labels out of range, "the codes may fit", total characters
enum { I_KIND, I_BYTES, I_P, I_M, I_BAD, I_CODES, I_CHARS, I_WORDS = 8 };
constexpr int KIND_CODES = 1, KIND_MAP = 2, KIND_NONE_FITS = 3;

// ape_label_rle_pack_dev: the map's H x W is the output size of the device size row dims (clamped to [1, cap]); the host's H and W
// are then the capacity, which sizes the grids and the workspace
__device__ __forceinline__ void dev_map_size(const int *dims, int cap, int &H, int &W) {
  if (!dims) return;
  const DevSizes d = dev_sizes(dims, 1, 1, cap);
  H = d.oh;
  W = d.ow;
}

// boundaries per column and the labels present (a run starts at every first occurrence of a label in column-major order).
// Labels outside [0, nlab) are flagged in info[I_BAD] and left out of the bitmap.
__global__ void __launch_bounds__(256) lrle_columns_kernel(const long long *__restrict__ L, int H, int W, int nlab,
                                                           uint32_t *__restrict__ present, int *__restrict__ colb,
                                                           int *__restrict__ info, const int *__restrict__ dims, int cap) {
  pdl_prologue();
  dev_map_size(dims, cap, H, W);
  const int lane = threadIdx.x & 31;
  const int x = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (x >= W) return;
  long long carry = x > 0 ? __ldg(L + (size_t)(H - 1) * W + x - 1) : 0;
  int nb = 0;
  bool bad = false;
  for (int y0 = 0; y0 < H; y0 += 32) {
    const int y = y0 + lane;
    const bool valid = y < H;
    const long long cur = valid ? __ldg(L + (size_t)y * W + x) : 0;
    long long prev = __shfl_up_sync(FULL, cur, 1);
    bool has_prev = true;
    if (lane == 0) {
      prev = carry;
      has_prev = x > 0 || y0 > 0;
    }
    const bool start = valid && (!has_prev || cur != prev);
    if (valid && (cur < 0 || cur >= nlab)) bad = true;
    else if (start) atomicOr(present + (cur >> 5), 1u << (cur & 31));
    nb += __popc(__ballot_sync(FULL, start && has_prev));
    carry = __shfl_sync(FULL, cur, 31);  // lane 31 is a pixel whenever another window follows
  }
  if (__any_sync(FULL, bad) && lane == 0) atomicOr(info + I_BAD, 1);
  if (lane == 0) colb[x] = nb;
}

// One CTA: index_of[label] = rank of each present label, label_of[rank] = label (rank < p_cap), P, m, and whether a codes body
// of at least 12 P + (2 m + 1 + P) bytes fits `cap`.  sizes (optional) <- P, m, labels out of range.
__global__ void __launch_bounds__(256) lrle_compact_kernel(const uint32_t *__restrict__ present, const int *__restrict__ colb, int W,
                                                           int p_cap, long long cap, int *__restrict__ index_of,
                                                           int *__restrict__ label_of, int *__restrict__ info, int *__restrict__ sizes,
                                                           const int *__restrict__ dims, int size_cap) {
  pdl_prologue();
  int H = 0;
  dev_map_size(dims, size_cap, H, W);
  __shared__ int s_warp[8];
  constexpr int PER = LRLE_WORDS / 256;
  uint32_t w[PER];
  int c = 0;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    w[i] = present[threadIdx.x * PER + i];
    c += __popc(w[i]);
  }
  int P;
  int r = block_excl_scan_256(c, s_warp, &P);
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    for (uint32_t b = w[i]; b; b &= b - 1) {
      const int label = (threadIdx.x * PER + i) * 32 + __ffs(b) - 1;
      index_of[label] = r;
      if (r < p_cap) label_of[r] = label;
      ++r;
    }
  }
  int part = 0;
  for (int x = threadIdx.x; x < W; x += 256) part += colb[x];
  int m;
  block_excl_scan_256(part, s_warp, &m);
  if (threadIdx.x == 0) {
    const int bad = info[I_BAD];
    const long long counts = 2LL * m + 1 + P;
    info[I_P] = P;
    info[I_M] = m;
    info[I_CODES] = !bad && P <= p_cap && 12LL * P + counts <= cap;
    if (sizes) {
      sizes[0] = P;
      sizes[1] = m;
      sizes[2] = bad;
    }
  }
}

// events per (present label, column): the label that starts and, after t = 0, the label that ends at every boundary
__global__ void __launch_bounds__(256) lrle_count_kernel(const long long *__restrict__ L, int H, int W, const int *__restrict__ index_of,
                                                         int *__restrict__ cnt, const int *__restrict__ info,
                                                         const int *__restrict__ dims, int cap) {
  pdl_prologue();
  if (!info[I_CODES]) return;
  dev_map_size(dims, cap, H, W);
  const int lane = threadIdx.x & 31;
  const int x = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (x >= W) return;
  long long carry = x > 0 ? __ldg(L + (size_t)(H - 1) * W + x - 1) : 0;
  for (int y0 = 0; y0 < H; y0 += 32) {
    const int y = y0 + lane;
    const bool valid = y < H;
    const long long cur = valid ? __ldg(L + (size_t)y * W + x) : 0;
    long long prev = __shfl_up_sync(FULL, cur, 1);
    bool has_prev = true;
    if (lane == 0) {
      prev = carry;
      has_prev = x > 0 || y0 > 0;
    }
    if (valid && (!has_prev || cur != prev)) {
      atomicAdd(cnt + (size_t)__ldg(index_of + cur) * W + x, 1);
      if (has_prev) atomicAdd(cnt + (size_t)__ldg(index_of + prev) * W + x, 1);
    }
    carry = __shfl_sync(FULL, cur, 31);
  }
}

// ---- exclusive scan of n ints in place, in three launches (tile sums, scan of the tile sums, tiles) -------------------------
__global__ void __launch_bounds__(256) lrle_scan_tiles_kernel(const int *__restrict__ data, long long n, int *__restrict__ sums,
                                                              const int *__restrict__ run) {
  pdl_prologue();
  if (!*run) return;
  __shared__ int s_warp[8];
  const long long base = (long long)blockIdx.x * LRLE_TILE + threadIdx.x * LRLE_ITEMS;
  int v = 0;
#pragma unroll
  for (int i = 0; i < LRLE_ITEMS; ++i) v += base + i < n ? data[base + i] : 0;
  int total;
  block_excl_scan_256(v, s_warp, &total);
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(256) lrle_scan_top_kernel(int *__restrict__ sums, int tiles, int *__restrict__ total,
                                                            const int *__restrict__ run) {
  pdl_prologue();
  if (!*run) return;
  __shared__ int s_warp[8];
  int base = 0;
  for (int i0 = 0; i0 < tiles; i0 += 256) {
    const int i = i0 + threadIdx.x;
    const int v = i < tiles ? sums[i] : 0;
    int sum;
    const int off = block_excl_scan_256(v, s_warp, &sum);
    if (i < tiles) sums[i] = base + off;
    base += sum;
  }
  if (total && threadIdx.x == 0) *total = base;
}

__global__ void __launch_bounds__(256) lrle_scan_apply_kernel(int *__restrict__ data, long long n, const int *__restrict__ sums,
                                                              const int *__restrict__ run) {
  pdl_prologue();
  if (!*run) return;
  __shared__ int s_warp[8];
  const long long base = (long long)blockIdx.x * LRLE_TILE + threadIdx.x * LRLE_ITEMS;
  int v[LRLE_ITEMS], t = 0;
#pragma unroll
  for (int i = 0; i < LRLE_ITEMS; ++i) {
    v[i] = base + i < n ? data[base + i] : 0;
    t += v[i];
  }
  int total;
  int off = sums[blockIdx.x] + block_excl_scan_256(t, s_warp, &total);
#pragma unroll
  for (int i = 0; i < LRLE_ITEMS; ++i) {
    if (base + i < n) data[base + i] = off;
    off += v[i];
  }
}

// Each event's position t, written at its (label, column) offset plus its rank among the label's events earlier in the column.
// off [P, W] holds the scanned offsets and is advanced as a cursor: afterwards off[p][W - 1] is the end of label p's positions.
// In a window of 32 pixels, mc = the lanes whose pixel has lane i's label c; the events of c in the window are the lanes where
// membership in mc changes (the pixel before the window counts as a member when it has label c), so an event's rank is the
// number of such changes at lower lanes.  A label that ends at lane i is the label of lane i - 1: its mask comes from there.
__global__ void __launch_bounds__(256) lrle_positions_kernel(const long long *__restrict__ L, int H, int W,
                                                             const int *__restrict__ index_of, int *__restrict__ off,
                                                             int *__restrict__ pos, const int *__restrict__ info,
                                                             const int *__restrict__ dims, int cap) {
  pdl_prologue();
  if (!info[I_CODES]) return;
  dev_map_size(dims, cap, H, W);
  const int lane = threadIdx.x & 31;
  const int x = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (x >= W) return;
  const unsigned lt = (1u << lane) - 1u;
  int cp = x > 0 ? __ldg(index_of + __ldg(L + (size_t)(H - 1) * W + x - 1)) : -1;  // label before the window (-1: none)
  for (int y0 = 0; y0 < H; y0 += 32) {
    const int y = y0 + lane;
    const bool valid = y < H;
    const unsigned vmask = __ballot_sync(FULL, valid);
    const int c = valid ? __ldg(index_of + __ldg(L + (size_t)y * W + x)) : -2;
    int a = __shfl_up_sync(FULL, c, 1);
    if (lane == 0) a = cp;
    const unsigned mc = __match_any_sync(FULL, c) & vmask;
    const unsigned tc = (mc ^ ((mc << 1) | (cp == c ? 1u : 0u))) & vmask;
    const unsigned mcp = __ballot_sync(FULL, valid && c == cp);
    unsigned ma = __shfl_up_sync(FULL, mc, 1);
    if (lane == 0) ma = mcp;
    const unsigned ta = (ma ^ ((ma << 1) | (cp == a ? 1u : 0u))) & vmask;
    if (valid && c != a) {
      const int t = x * H + y;
      pos[off[(size_t)c * W + x] + __popc(tc & lt)] = t;
      if (a >= 0) pos[off[(size_t)a * W + x] + __popc(ta & lt)] = t;
    }
    __syncwarp();
    // the lowest lane of each label advances its cursor; lane 0 that of a carried label absent from the window
    if (valid && (mc & lt) == 0) off[(size_t)c * W + x] += __popc(tc);
    if (lane == 0 && cp >= 0 && mcp == 0) off[(size_t)cp * W + x] += __popc(ta);
    __syncwarp();
    cp = __shfl_sync(FULL, c, 31);
  }
}

// count g of the codes body: label p, and the value rleToString codes, i.e. count i of p (the differences of [0, positions of
// p..., H * W]) minus count i - 2 from the fourth on.  Count g belongs to p when start(p) + p <= g < start(p + 1) + p + 1.
__device__ __forceinline__ long long lrle_value(int g, const int *__restrict__ off, int W, int P, const int *__restrict__ pos,
                                                long long HW, int *label_p) {
  auto start = [&](int p) { return p > 0 ? off[(size_t)p * W - 1] : 0; };  // end of label p - 1 = off[p - 1][W - 1]
  int lo = 0, hi = P - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (start(mid) + mid <= g) lo = mid;
    else hi = mid - 1;
  }
  const int s = start(lo), e = off[(size_t)lo * W + W - 1], i = g - s - lo;
  auto at = [&](int j) -> long long { return j < 0 ? 0 : j >= e - s ? HW : (long long)pos[s + j]; };
  long long x = at(i) - at(i - 1);
  if (i > 2) x -= at(i - 2) - at(i - 3);
  *label_p = lo;
  return x;
}

// LEN: clen[g] = characters of count g (0 past the last count).  Otherwise, when the state says the codes fit: the characters
// at body + 12 P + clen[g] (clen scanned), and thread g < P writes label g's table row.
template <bool LEN>
__global__ void __launch_bounds__(256) lrle_chars_kernel(const int *__restrict__ off, int W, const int *__restrict__ pos, long long HW,
                                                         int *__restrict__ clen, long long ncap, const int *__restrict__ label_of,
                                                         const int *__restrict__ info, uint8_t *__restrict__ body,
                                                         const int *__restrict__ dims, int cap) {
  pdl_prologue();
  if (LEN ? !info[I_CODES] : info[I_KIND] != KIND_CODES) return;
  if (dims) {
    int H = 0;
    dev_map_size(dims, cap, H, W);
    HW = (long long)H * W;
  }
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= ncap) return;
  const int P = info[I_P];
  const long long counts = 2LL * info[I_M] + 1 + P;
  if (!LEN && g < P) {
    auto first = [&](int p) -> long long { return p > 0 ? off[(size_t)p * W - 1] + p : 0; };  // index of label p's first count
    const int o = clen[first((int)g)];
    const int end = g + 1 < P ? clen[first((int)g + 1)] : info[I_CHARS];
    int *row = reinterpret_cast<int *>(body) + 3 * g;
    row[0] = __ldg(label_of + g);
    row[1] = o;
    row[2] = end - o;
  }
  if (g >= counts) {
    if (LEN) clen[g] = 0;
    return;
  }
  int p;
  const long long x = lrle_value((int)g, off, W, P, pos, HW, &p);
  if (LEN) clen[g] = rle_chars(x, nullptr, 0);
  else rle_chars(x, body + 12LL * P + clen[g], 7);
}

// kind, bytes and P of the result; a codes body that turned out longer than cap falls back to the map (2 H W bytes) if that
// fits, else nothing fits: bytes is then the smaller of the two forms (a lower bound for codes that were not built)
__global__ void lrle_finalize_kernel(int *__restrict__ info, long long HW, long long cap, int map_ok, int *__restrict__ out_info,
                                     const int *__restrict__ dims, int size_cap) {
  pdl_prologue();
  if (dims) {
    int H = 0, W = 0;
    dev_map_size(dims, size_cap, H, W);
    HW = (long long)H * W;
  }
  const long long P = info[I_P], codes_min = 12 * P + 2LL * info[I_M] + 1 + P;
  const long long codes = info[I_CODES] ? 12 * P + info[I_CHARS] : codes_min;
  int kind, bytes;
  if (info[I_CODES] && codes <= cap) {
    kind = KIND_CODES;
    bytes = (int)codes;
  } else if (map_ok && !info[I_BAD] && 2 * HW <= cap) {
    kind = KIND_MAP;
    bytes = (int)(2 * HW);
  } else {
    kind = KIND_NONE_FITS;
    bytes = info[I_BAD] ? 0 : (int)min(min(codes, 2 * HW), 0x7fffffffLL);
  }
  info[I_KIND] = kind;
  info[I_BYTES] = bytes;
  out_info[0] = kind;
  out_info[1] = bytes;
  out_info[2] = (int)P;
}

// the map as uint16, row-major, when the slot holds it
__global__ void __launch_bounds__(256) lrle_map_kernel(const long long *__restrict__ L, long long HW, const int *__restrict__ info,
                                                       uint16_t *__restrict__ out, const int *__restrict__ dims, int cap) {
  pdl_prologue();
  if (info[I_KIND] != KIND_MAP) return;
  if (dims) {
    int H = 0, W = 0;
    dev_map_size(dims, cap, H, W);
    HW = (long long)H * W;
  }
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < HW) out[i] = (uint16_t)__ldg(L + i);
}

// workspace, every part 256-byte aligned: the bitmap and the state block first (ape_label_rle_sizes uses only the parts that do
// not depend on P), then [p_cap, W] counts / offsets, ev_cap positions and ev_cap + p_cap character lengths / offsets
struct LrleWs {
  uint32_t *present;
  int *index_of, *info, *colb, *label_of, *off, *pos, *clen, *sums;
  long long ncap;
  int64_t bytes;
};

long long lrle_tiles(long long n) { return (n + LRLE_TILE - 1) / LRLE_TILE; }

LrleWs lrle_ws(void *base, int W, int p_cap, long long ev_cap) {
  LrleWs w{};
  int64_t o = 0;
  auto take = [&](int64_t n) {
    const int64_t at = o;
    o += (n + 255) / 256 * 256;
    return reinterpret_cast<char *>(reinterpret_cast<uintptr_t>(base) + at);
  };
  w.present = reinterpret_cast<uint32_t *>(take(4LL * LRLE_WORDS));
  w.info = reinterpret_cast<int *>(take(4LL * I_WORDS));
  w.index_of = reinterpret_cast<int *>(take(4LL * LRLE_LABELS));
  w.colb = reinterpret_cast<int *>(take(4LL * W));
  w.ncap = ev_cap + p_cap;
  w.label_of = reinterpret_cast<int *>(take(4LL * p_cap));
  w.off = reinterpret_cast<int *>(take(4LL * p_cap * W));
  w.pos = reinterpret_cast<int *>(take(4LL * ev_cap));
  w.clen = reinterpret_cast<int *>(take(4LL * w.ncap));
  w.sums = reinterpret_cast<int *>(take(4LL * std::max(std::max(lrle_tiles((long long)p_cap * W), lrle_tiles(w.ncap)), 1LL)));
  w.bytes = o;
  return w;
}

int lrle_scan(int *data, long long n, int *sums, int *total, const int *run, cudaStream_t st) {
  const long long tiles = lrle_tiles(n);
  if (tiles == 0) return APE_OK;
  int rc;
  APE_LAUNCH(lrle_scan_tiles_kernel, tiles, 256, 0, st, (const int *)data, n, sums, run);
  if ((rc = check_launch("lrle_scan_tiles_kernel"))) return rc;
  APE_LAUNCH(lrle_scan_top_kernel, 1, 256, 0, st, sums, (int)tiles, total, run);
  if ((rc = check_launch("lrle_scan_top_kernel"))) return rc;
  APE_LAUNCH(lrle_scan_apply_kernel, tiles, 256, 0, st, data, n, (const int *)sums, run);
  return check_launch("lrle_scan_apply_kernel");
}

// the first two passes (bitmap, boundaries, compaction); the state block says whether the rest runs
int lrle_front(const long long *L, int H, int W, int nlab, int p_cap, long long cap, const LrleWs &ws, int *sizes, cudaStream_t st,
               const int *dims = nullptr) {
  cudaError_t e = cudaMemsetAsync(ws.present, 0, 4LL * LRLE_WORDS, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(ws.info, 0, 4LL * I_WORDS, st);
  if (e != cudaSuccess) return fail((int)e, "label_rle: %s", cudaGetErrorString(e));
  int rc;
  APE_LAUNCH(lrle_columns_kernel, (W + 7) / 8, 256, 0, st, L, H, W, nlab, ws.present, ws.colb, ws.info, dims, W);
  if ((rc = check_launch("lrle_columns_kernel"))) return rc;
  APE_LAUNCH(lrle_compact_kernel, 1, 256, 0, st, (const uint32_t *)ws.present, (const int *)ws.colb, W, p_cap, cap, ws.index_of,
             ws.label_of, ws.info, sizes, dims, W);
  return check_launch("lrle_compact_kernel");
}

// everything after lrle_front: the codes body at `body` if it fits cap, else (map != NULL) the map as uint16 if that fits
int lrle_rest(const long long *L, int H, int W, int p_cap, long long cap, const LrleWs &ws, uint8_t *body, uint16_t *map, int *out_info,
              cudaStream_t st, const int *dims = nullptr) {
  const long long HW = (long long)H * W;
  const int *run = ws.info + I_CODES;
  cudaError_t e = cudaMemsetAsync(ws.off, 0, 4LL * p_cap * W, st);
  if (e != cudaSuccess) return fail((int)e, "label_rle: %s", cudaGetErrorString(e));
  int rc;
  const int col_blocks = (W + 7) / 8;
  APE_LAUNCH(lrle_count_kernel, col_blocks, 256, 0, st, L, H, W, (const int *)ws.index_of, ws.off, (const int *)ws.info, dims, W);
  if ((rc = check_launch("lrle_count_kernel"))) return rc;
  if ((rc = lrle_scan(ws.off, (long long)p_cap * W, ws.sums, nullptr, run, st))) return rc;
  APE_LAUNCH(lrle_positions_kernel, col_blocks, 256, 0, st, L, H, W, (const int *)ws.index_of, ws.off, ws.pos, (const int *)ws.info, dims, W);
  if ((rc = check_launch("lrle_positions_kernel"))) return rc;
  const long long blocks = (ws.ncap + 255) / 256;
  APE_LAUNCH((lrle_chars_kernel<true>), blocks, 256, 0, st, (const int *)ws.off, W, (const int *)ws.pos, HW, ws.clen, ws.ncap,
             (const int *)ws.label_of, (const int *)ws.info, body, dims, W);
  if ((rc = check_launch("lrle_chars_kernel"))) return rc;
  if ((rc = lrle_scan(ws.clen, ws.ncap, ws.sums, ws.info + I_CHARS, run, st))) return rc;
  APE_LAUNCH(lrle_finalize_kernel, 1, 1, 0, st, ws.info, HW, cap, map ? 1 : 0, out_info, dims, W);
  if ((rc = check_launch("lrle_finalize_kernel"))) return rc;
  APE_LAUNCH((lrle_chars_kernel<false>), blocks, 256, 0, st, (const int *)ws.off, W, (const int *)ws.pos, HW, ws.clen, ws.ncap,
             (const int *)ws.label_of, (const int *)ws.info, body, dims, W);
  if ((rc = check_launch("lrle_chars_kernel"))) return rc;
  if (map) {
    APE_LAUNCH(lrle_map_kernel, (HW + 255) / 256, 256, 0, st, L, HW, (const int *)ws.info, map, dims, W);
    if ((rc = check_launch("lrle_map_kernel"))) return rc;
  }
  return APE_OK;
}

bool lrle_geometry_ok(int H, int W) { return H > 0 && W > 0 && (long long)H * W <= (1LL << 27); }

}  // namespace
}  // namespace ape

using namespace ape;

extern "C" int64_t ape_label_rle_workspace_bytes(int W, int P, int64_t events) {
  if (W <= 0 || P < 0 || P > LRLE_LABELS || events < 0) return 0;
  return lrle_ws(nullptr, W, P, events).bytes;
}

extern "C" int ape_label_rle_sizes(const int64_t *label, int H, int W, void *workspace, int *sizes, void *stream) {
  if (!label || !workspace || !sizes) return fail(APE_ERR_NULL_PTR, "label_rle_sizes: null pointer");
  if (!lrle_geometry_ok(H, W)) return fail(APE_ERR_INVALID_ARG, "label_rle_sizes: bad map size %dx%d (at most 2^27 pixels)", H, W);
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(APE_ERR_INVALID_ARG, "label_rle_sizes: workspace must be 256-byte aligned");
  const LrleWs ws = lrle_ws(workspace, W, 0, 0);
  return lrle_front((const long long *)label, H, W, LRLE_LABELS, 0, 0, ws, sizes, (cudaStream_t)stream);
}

extern "C" int64_t ape_label_rle_out_bytes(int P, int m) {
  if (P < 0 || m < 0) return 0;
  return 12LL * P + 7LL * (2LL * m + 1 + P);
}

extern "C" int ape_label_rle(const int64_t *label, int H, int W, const int *sizes, void *workspace, uint8_t *out, int *out_info,
                             void *stream) {
  if (!label || !sizes || !workspace || !out || !out_info) return fail(APE_ERR_NULL_PTR, "label_rle: null pointer");
  if (!lrle_geometry_ok(H, W)) return fail(APE_ERR_INVALID_ARG, "label_rle: bad map size %dx%d (at most 2^27 pixels)", H, W);
  const int P = sizes[0], m = sizes[1];
  if (sizes[2]) return fail(APE_ERR_INVALID_ARG, "label_rle: labels outside [0, 65535]");
  if (P < 1 || P > LRLE_LABELS || m < 0 || (long long)m >= (long long)H * W)
    return fail(APE_ERR_INVALID_ARG, "label_rle: sizes P=%d m=%d do not describe a %dx%d map", P, m, H, W);
  if ((reinterpret_cast<uintptr_t>(workspace) & 255) || (reinterpret_cast<uintptr_t>(out) & 3))
    return fail(APE_ERR_INVALID_ARG, "label_rle: workspace must be 256-byte and out 4-byte aligned");
  const long long events = 2LL * m + 1, cap = ape_label_rle_out_bytes(P, m);
  const LrleWs ws = lrle_ws(workspace, W, P, events);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = lrle_front((const long long *)label, H, W, LRLE_LABELS, P, cap, ws, nullptr, st);
  if (rc) return rc;
  return lrle_rest((const long long *)label, H, W, P, cap, ws, out, nullptr, out_info, st);
}

namespace {
int lrle_pack_caps(int num_labels, int slot, int *p_cap) {
  *p_cap = std::min(num_labels, slot / 13);  // 12 bytes of table and at least one character per present label
  return slot;                               // every event is a count of at least one character
}
}  // namespace

extern "C" int64_t ape_label_rle_pack_workspace_bytes(int W, int num_labels, int slot) {
  if (W <= 0 || num_labels <= 0 || num_labels > LRLE_LABELS || slot <= 0) return 0;
  int p_cap;
  const int ev_cap = lrle_pack_caps(num_labels, slot, &p_cap);
  return lrle_ws(nullptr, W, p_cap, ev_cap).bytes;
}

extern "C" int ape_label_rle_pack(const int64_t *label, int H, int W, int num_labels, int slot, void *workspace, uint8_t *out,
                                  int *out_info, void *stream) {
  if (!label || !workspace || !out || !out_info) return fail(APE_ERR_NULL_PTR, "label_rle_pack: null pointer");
  if (!lrle_geometry_ok(H, W)) return fail(APE_ERR_INVALID_ARG, "label_rle_pack: bad map size %dx%d (at most 2^27 pixels)", H, W);
  if (num_labels <= 0 || num_labels > LRLE_LABELS)
    return fail(APE_ERR_INVALID_ARG, "label_rle_pack: num_labels %d outside [1, 65536]", num_labels);
  if (slot < 16 || slot % 4 != 0) return fail(APE_ERR_INVALID_ARG, "label_rle_pack: slot of %d bytes (a multiple of 4, >= 16)", slot);
  if ((reinterpret_cast<uintptr_t>(workspace) & 255) || (reinterpret_cast<uintptr_t>(out) & 3))
    return fail(APE_ERR_INVALID_ARG, "label_rle_pack: workspace must be 256-byte and out 4-byte aligned");
  int p_cap;
  const int ev_cap = lrle_pack_caps(num_labels, slot, &p_cap);
  const LrleWs ws = lrle_ws(workspace, W, p_cap, ev_cap);
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(out, 0, slot, st);
  if (e != cudaSuccess) return fail((int)e, "label_rle_pack: %s", cudaGetErrorString(e));
  int rc = lrle_front((const long long *)label, H, W, num_labels, p_cap, slot, ws, nullptr, st);
  if (rc) return rc;
  return lrle_rest((const long long *)label, H, W, p_cap, slot, ws, out, reinterpret_cast<uint16_t *>(out), out_info, st);
}

extern "C" int ape_label_rle_pack_dev(const int64_t *label, const int *sizes, int cap, int num_labels, int slot, void *workspace,
                                      uint8_t *out, int *out_info, void *stream) {
  if (!label || !sizes || !workspace || !out || !out_info) return fail(APE_ERR_NULL_PTR, "label_rle_pack_dev: null pointer");
  if (!lrle_geometry_ok(cap, cap))
    return fail(APE_ERR_INVALID_ARG, "label_rle_pack_dev: capacity %d (at most 2^27 pixels in a capacity x capacity map)", cap);
  if (num_labels <= 0 || num_labels > LRLE_LABELS)
    return fail(APE_ERR_INVALID_ARG, "label_rle_pack_dev: num_labels %d outside [1, 65536]", num_labels);
  if (slot < 16 || slot % 4 != 0) return fail(APE_ERR_INVALID_ARG, "label_rle_pack_dev: slot of %d bytes (a multiple of 4, >= 16)", slot);
  if ((reinterpret_cast<uintptr_t>(workspace) & 255) || (reinterpret_cast<uintptr_t>(out) & 3))
    return fail(APE_ERR_INVALID_ARG, "label_rle_pack_dev: workspace must be 256-byte and out 4-byte aligned");
  int p_cap;
  const int ev_cap = lrle_pack_caps(num_labels, slot, &p_cap);
  const LrleWs ws = lrle_ws(workspace, cap, p_cap, ev_cap);
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(out, 0, slot, st);
  if (e != cudaSuccess) return fail((int)e, "label_rle_pack_dev: %s", cudaGetErrorString(e));
  int rc = lrle_front((const long long *)label, cap, cap, num_labels, p_cap, slot, ws, nullptr, st, sizes);
  if (rc) return rc;
  return lrle_rest((const long long *)label, cap, cap, p_cap, slot, ws, out, reinterpret_cast<uint16_t *>(out), out_info, st, sizes);
}
