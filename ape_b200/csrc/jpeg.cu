// jpeg.cu — sequential-JPEG decode on the device, bit for bit with Pillow (libjpeg's default settings), DESIGN.md §4.16.
//
// The host walks the markers (ape_b200/jpeg.py) and uploads the entropy-coded scan with the Huffman lookup tables, the
// quantisation tables and, with restart markers, the offset of each restart interval.  Then, on one stream:
//
//   huffman     sequential Huffman decode (ITU-T T.81 F.2.2) into quantised int16 coefficients, natural order, one block of 64
//               per 8x8 block in MCU order; DC predictions turned into absolute values on the way.
//                 * restart interval > 0: one thread per interval (T.81 F.2.1.3.1: every interval starts byte-aligned with
//                   zero predictions), huff_write_kernel alone.
//                 * no restart interval (Pillow's default): self-synchronising parallel decoding over fixed subsequences of
//                   SUBSEQ_BYTES bytes (Weissenberger & Schmidt, ICPP 2018), with the decoder state of the JPEG variant:
//                   (bit position, block of the MCU, zig-zag index).  huff_spec_kernel decodes every subsequence from a guessed
//                   entry state (block 0, index 0, at the subsequence's first byte) to the first codeword boundary at or
//                   past its end; huff_prop_kernel re-decodes each subsequence whose guess differs from its predecessor's exit;
//                   huff_chain_kernel (one warp) walks the exits in order, re-decodes the rare subsequence that is still out of
//                   step (so the result never depends on synchronisation happening), and takes the prefix sums of the block
//                   counts and per-component DC sums; huff_write_kernel decodes each subsequence once more from its true
//                   entry, writing coefficients at the block its prefix names with absolute DC values.
//   idct        dequantise + JDCT_ISLOW per block (8 threads per block, the column pass through shared memory), into one
//               uint8 plane per component covering whole MCUs.
//   colour      one thread per output pixel, at its final orientation: the EXIF transpose (detectron2 _apply_exif_orientation),
//               libjpeg's fancy chroma upsampling, the fixed-point YCbCr -> RGB, the channel order; grayscale replicated.
//
// Stuffed 0x00 bytes (T.81 F.1.2.3) are dropped by the bit reader as it fetches bytes.  Bit positions are counted in the
// unstuffed stream relative to the byte a decoder starts at; the exit state of a subsequence is stored relative to the first
// byte of the next one, so two decoders compare positions without a global prefix over the stuffing.  Reads stop at the scan
// length (zeros beyond, never an out-of-range load); a needed codeword that runs past the end, an invalid code, or fewer
// blocks than the frame needs set a bit of the device status word (ape_jpeg_status_error turns it into ape_last_error()).
#include "common.cuh"

namespace ape {
namespace {

constexpr int TABLE_WORDS = 1024;  // one Huffman table as uploaded by ape_b200/jpeg.py huffman_lut()
constexpr int LUT_BITS = 9, MAXCODE_OFF = 512, VALOFF_OFF = 529, VALS_OFF = 546;
constexpr int MAX_TABLES = 6;
constexpr int SUBSEQ_BYTES = 512;
constexpr int DEC_THREADS = 128;

enum : int { ERR_BAD_CODE = 1, ERR_TRUNCATED = 2, ERR_SHORT = 4 };

// T.81 Figure A.6; entries 64..79 repeat 63 so that a run pushing the index past 63 lands on the last coefficient, as libjpeg's
// extended jpeg_natural_order does for corrupt data
__constant__ uint8_t kNatural[80] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
    6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
    39, 46, 53, 60, 61, 54, 47, 55, 62, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63};

struct Geom {
  int ncomp, bpm, mx, my, width, height, n_blocks, scan_bytes;
  int hmax, vmax, dw, dh;                  // chroma samples per row / rows (the downsampled width and height)
  int blk_comp[6], blk_dy[6], blk_dx[6];   // component and position of each block of an MCU
  int comp_h[3], comp_v[3], dc_tab[3], ac_tab[3], q_tab[3];
  int plane_w[3], plane_h[3];
  long long plane_off[3];
  int restart_interval, n_intervals, n_sub, orientation, bgr;
};

// ---- bit reader ------------------------------------------------------------------------------------------------------
struct BitReader {
  const uint8_t *p;
  int idx, end;          // next byte to fetch, fetch limit (zeros beyond)
  unsigned prev;         // last byte fetched (a 0x00 after 0xFF is stuffing)
  unsigned long long acc;  // unconsumed bits, MSB first
  int nbits;
  long long consumed;    // unstuffed bits consumed since the start byte
  long long real_bits;   // unstuffed bits before `end` from the start byte (known once the fetch reaches `end`)

  __device__ __forceinline__ void init(const uint8_t *data, int start, int limit) {
    p = data;
    idx = start;
    end = limit;
    prev = start > 0 ? __ldg(data + start - 1) : 0u;
    acc = 0;
    nbits = 0;
    consumed = 0;
    real_bits = 1ll << 62;
  }
  __device__ __forceinline__ void refill() {  // afterwards nbits >= 57: one codeword (<= 16) + its value bits (<= 15)
    while (nbits <= 56) {
      if (idx < end) {
        const unsigned b = __ldg(p + idx);
        const bool stuffed = b == 0u && prev == 0xFFu;
        prev = b;
        ++idx;
        if (stuffed) continue;
        acc |= (unsigned long long)b << (56 - nbits);
      } else if (real_bits == (1ll << 62)) {
        real_bits = consumed + nbits;
      }
      nbits += 8;
    }
  }
  __device__ __forceinline__ unsigned peek(int n) const { return (unsigned)(acc >> (64 - n)); }
  __device__ __forceinline__ void skip(int n) {
    acc <<= n;
    nbits -= n;
    consumed += n;
  }
  __device__ __forceinline__ int get(int n) {  // n in 0..16
    if (n == 0) return 0;
    const int v = (int)peek(n);
    skip(n);
    return v;
  }
};

// T.81 F.2.2.1 EXTEND
__device__ __forceinline__ int extend(int v, int s) { return (s != 0 && v < (1 << (s - 1))) ? v - (1 << s) + 1 : v; }

// T.81 F.2.2.3 DECODE: a 9-bit table read resolves codes of <= 9 bits; longer codes compare against MAXCODE per length.  An
// invalid code (none of 16 bits matches: the all-ones prefix) reads as symbol 0 after 16 bits and raises `bad`.
__device__ __forceinline__ int decode_symbol(BitReader &br, const int *tab, bool &bad) {
  const int e = tab[br.peek(LUT_BITS)];
  if (e != 0) {
    br.skip(e >> 8);
    return e & 255;
  }
  const unsigned code16 = br.peek(16);
#pragma unroll 1
  for (int l = LUT_BITS + 1; l <= 16; ++l) {
    const int code = (int)(code16 >> (16 - l));
    if (code <= tab[MAXCODE_OFF + l]) {
      br.skip(l);
      return tab[VALS_OFF + tab[VALOFF_OFF + l] + code];
    }
  }
  bad = true;
  br.skip(16);
  return 0;
}

struct Run {
  int c, k;             // block of the MCU, zig-zag index (0 = the next symbol is a DC difference)
  long long block;      // index of the block being decoded (MCU order), -1 before the first
  int dc[3];            // DC prediction per component (or the sum of differences, for a guessed entry)
  bool bad;
};

// Decode codewords while the position is before stop_bits and fewer than max_blocks blocks have been started.  WRITE: store
// each coefficient (DC as its absolute value) into coef; error bits go to status.
template <bool WRITE>
__device__ void decode_run(BitReader &br, const int *tabs, const Geom &g, Run &r, long long stop_bits, long long max_blocks,
                           int16_t *coef) {
#pragma unroll 1
  while (br.consumed < stop_bits) {
    if (r.k == 0 && r.block + 1 >= max_blocks) break;
    br.refill();
    const int comp = g.blk_comp[r.c];
    if (r.k == 0) {
      const int s = decode_symbol(br, tabs + g.dc_tab[comp] * TABLE_WORDS, r.bad);
      const int v = extend(br.get(s), s);
      // the component picked by selects rather than an index, so the predictions stay in registers
      const int d = (comp == 0 ? r.dc[0] : comp == 1 ? r.dc[1] : r.dc[2]) + v;
      r.dc[0] = comp == 0 ? d : r.dc[0];
      r.dc[1] = comp == 1 ? d : r.dc[1];
      r.dc[2] = comp == 2 ? d : r.dc[2];
      ++r.block;
      r.k = 1;
      if (WRITE) coef[r.block * 64] = (int16_t)d;
    } else {
      const int rs = decode_symbol(br, tabs + g.ac_tab[comp] * TABLE_WORDS, r.bad);
      const int run = rs >> 4, s = rs & 15;
      if (s != 0) {
        r.k += run;
        const int v = extend(br.get(s), s);
        if (WRITE) coef[r.block * 64 + kNatural[r.k]] = (int16_t)v;
        ++r.k;
      } else if (run == 15) {
        r.k += 16;
      } else {
        r.k = 64;  // EOB
      }
      if (r.k >= 64) {
        r.k = 0;
        r.c = r.c + 1 == g.bpm ? 0 : r.c + 1;
      }
    }
    if (WRITE && br.consumed > br.real_bits) break;  // a needed codeword ran past the data: reported by the caller
  }
}

__device__ __forceinline__ void load_tables(int *sh, const int *huff, int n_tables) {
  for (int i = threadIdx.x; i < n_tables * TABLE_WORDS; i += blockDim.x) sh[i] = __ldg(huff + i);
  __syncthreads();
}

// Unstuffed bits in [b0, b1) of the scan (b0's predecessor decides whether b0 itself is a stuffed byte).
__device__ long long unstuffed_bits(const uint8_t *scan, int b0, int b1) {
  int n = 0;
  unsigned prev = b0 > 0 ? __ldg(scan + b0 - 1) : 0u;
#pragma unroll 4
  for (int i = b0; i < b1; ++i) {
    const unsigned b = __ldg(scan + i);
    n += (b == 0u && prev == 0xFFu);
    prev = b;
  }
  return 8ll * (b1 - b0 - n);
}

// Decode subsequence t from entry e = (bit offset past its first byte, c, k); exit x relative to subsequence t+1's first
// byte; a = (blocks started, DC difference sums per component).
__device__ void spec_one(const uint8_t *scan, const int *tabs, const Geom &g, int t, int4 e, int4 &x, int4 &a) {
  const int b0 = t * SUBSEQ_BYTES, b1 = min(b0 + SUBSEQ_BYTES, g.scan_bytes);
  const long long end_bits = unstuffed_bits(scan, b0, b1);
  BitReader br;
  br.init(scan, b0, g.scan_bytes);
  br.refill();
  br.skip(e.x);
  Run r{e.y, e.z, -1, {0, 0, 0}, false};
  decode_run<false>(br, tabs, g, r, end_bits, 1ll << 62, nullptr);
  x = make_int4((int)(br.consumed - end_bits), r.c, r.k, 0);
  a = make_int4((int)(r.block + 1), r.dc[0], r.dc[1], r.dc[2]);
}

__global__ void __launch_bounds__(DEC_THREADS) huff_spec_kernel(const uint8_t *__restrict__ scan, const int *__restrict__ huff,
                                                                int n_tables, Geom g, int4 *E, int4 *X, int4 *A) {
  extern __shared__ int sh_tabs[];
  pdl_prologue();
  load_tables(sh_tabs, huff, n_tables);
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= g.n_sub) return;
  const int4 e = make_int4(0, 0, 0, 0);
  int4 x, a;
  spec_one(scan, sh_tabs, g, t, e, x, a);
  E[t] = e;
  X[t] = x;
  A[t] = a;
}

__device__ __forceinline__ bool same_state(int4 a, int4 b) { return a.x == b.x && a.y == b.y && a.z == b.z; }

__global__ void __launch_bounds__(DEC_THREADS) huff_prop_kernel(const uint8_t *__restrict__ scan, const int *__restrict__ huff,
                                                                int n_tables, Geom g, int4 *E, const int4 *X0, const int4 *A0,
                                                                int4 *X1, int4 *A1) {
  extern __shared__ int sh_tabs[];
  pdl_prologue();
  load_tables(sh_tabs, huff, n_tables);
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= g.n_sub) return;
  int4 x = X0[t], a = A0[t];
  if (t > 0) {
    const int4 prev = X0[t - 1];
    if (!same_state(prev, E[t])) {
      E[t] = prev;
      spec_one(scan, sh_tabs, g, t, prev, x, a);
    }
  }
  X1[t] = x;
  A1[t] = a;
}

// One warp: settle every entry state in order (re-decoding a subsequence whose entry differs from its predecessor's exit),
// then P[t] = (first block index, DC predictions per component) at each subsequence's entry.
__global__ void __launch_bounds__(32) huff_chain_kernel(const uint8_t *__restrict__ scan, const int *__restrict__ huff,
                                                        int n_tables, Geom g, int4 *E, const int4 *X, const int4 *A, int4 *P,
                                                        int *status) {
  extern __shared__ int sh_tabs[];
  pdl_prologue();
  load_tables(sh_tabs, huff, n_tables);
  const int lane = threadIdx.x;
  int4 carry_x = make_int4(0, 0, 0, 0);
  long long carry_blocks = 0;
  int carry_dc[3] = {0, 0, 0};
  for (int base = 0; base < g.n_sub; base += 32) {
    const int t = base + lane;
    int4 e = make_int4(0, 0, 0, 0), x = e, a = e;
    if (t < g.n_sub) {
      e = E[t];
      x = X[t];
      a = A[t];
    }
    bool fixed = false;
    for (;;) {
      int4 px;
      px.x = __shfl_up_sync(0xffffffffu, x.x, 1);
      px.y = __shfl_up_sync(0xffffffffu, x.y, 1);
      px.z = __shfl_up_sync(0xffffffffu, x.z, 1);
      if (lane == 0) px = carry_x;
      const bool mism = t < g.n_sub && t > 0 && !same_state(px, e);
      const unsigned bal = __ballot_sync(0xffffffffu, mism);
      if (bal == 0u) break;
      if (lane == __ffs(bal) - 1) {
        e = make_int4(px.x, px.y, px.z, 0);
        spec_one(scan, sh_tabs, g, t, e, x, a);
        fixed = true;
      }
      __syncwarp();
    }
    if (fixed) E[t] = e;
    // exclusive prefix of (blocks, dc sums) across the warp
    int blk = a.x, d0 = a.y, d1 = a.z, d2 = a.w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int b_ = __shfl_up_sync(0xffffffffu, blk, o), x0 = __shfl_up_sync(0xffffffffu, d0, o);
      const int x1 = __shfl_up_sync(0xffffffffu, d1, o), x2 = __shfl_up_sync(0xffffffffu, d2, o);
      if (lane >= o) {
        blk += b_;
        d0 += x0;
        d1 += x1;
        d2 += x2;
      }
    }
    if (t < g.n_sub)
      P[t] = make_int4((int)(carry_blocks + blk - a.x), carry_dc[0] + d0 - a.y, carry_dc[1] + d1 - a.z, carry_dc[2] + d2 - a.w);
    carry_blocks += __shfl_sync(0xffffffffu, blk, 31);
    carry_dc[0] += __shfl_sync(0xffffffffu, d0, 31);
    carry_dc[1] += __shfl_sync(0xffffffffu, d1, 31);
    carry_dc[2] += __shfl_sync(0xffffffffu, d2, 31);
    carry_x.x = __shfl_sync(0xffffffffu, x.x, 31);
    carry_x.y = __shfl_sync(0xffffffffu, x.y, 31);
    carry_x.z = __shfl_sync(0xffffffffu, x.z, 31);
  }
  if (lane == 0 && carry_blocks < g.n_blocks) atomicOr(status, ERR_SHORT);
}

// Subsequence mode: thread t decodes subsequence t from E[t] with the prefix P[t].  Restart mode: thread t
// decodes restart interval t from its first byte with zero predictions.
__global__ void __launch_bounds__(DEC_THREADS) huff_write_kernel(const uint8_t *__restrict__ scan, const int *__restrict__ huff,
                                                                 int n_tables, Geom g, const int4 *E, const int4 *P,
                                                                 int restart_mode, const int *__restrict__ rst, int16_t *coef,
                                                                 int *status) {
  extern __shared__ int sh_tabs[];
  pdl_prologue();
  load_tables(sh_tabs, huff, n_tables);
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  BitReader br;
  Run r;
  long long stop_bits, max_blocks;
  if (!restart_mode) {
    if (t >= g.n_sub) return;
    const int b0 = t * SUBSEQ_BYTES, b1 = min(b0 + SUBSEQ_BYTES, g.scan_bytes);
    stop_bits = unstuffed_bits(scan, b0, b1);
    const int4 e = E[t], p = P[t];
    br.init(scan, b0, g.scan_bytes);
    br.refill();
    br.skip(e.x);
    r = Run{e.y, e.z, (long long)p.x - 1, {p.y, p.z, p.w}, false};
    max_blocks = g.n_blocks;
  } else {
    if (t >= g.n_intervals) return;
    const int b0 = t == 0 ? 0 : __ldg(rst + t - 1);
    const int b1 = t + 1 < g.n_intervals ? __ldg(rst + t) - 2 : g.scan_bytes;
    br.init(scan, b0, b1);
    const long long mcu0 = (long long)t * g.restart_interval;
    const long long mcu1 = min(mcu0 + g.restart_interval, (long long)g.mx * g.my);
    r = Run{0, 0, mcu0 * g.bpm - 1, {0, 0, 0}, false};
    stop_bits = 1ll << 62;
    max_blocks = mcu1 * g.bpm;
  }
  decode_run<true>(br, sh_tabs, g, r, stop_bits, max_blocks, coef);
  int err = r.bad ? ERR_BAD_CODE : 0;
  if (br.consumed > br.real_bits) err |= ERR_TRUNCATED;
  if (restart_mode && r.block + 1 < max_blocks) err |= ERR_SHORT;
  if (err) atomicOr(status, err);
}

// ---- IDCT ------------------------------------------------------------------------------------------------------------
// JDCT_ISLOW (libjpeg's default): the Loeffler-Ligtenberg-Moschytz flow graph with 12 multiplications per 1-D transform,
// constants FIX(x) = round(x * 2^13); pass 1 (columns) keeps PASS1_BITS = 2 extra bits, pass 2 (rows) removes 13 + 2 + 3
// (the 1/8 of the 2-D normalisation), both descale by adding half and shifting right arithmetically; the result indexes the
// range-limit table with (value & 1023).  Arithmetic in 64 bits as libjpeg's JLONG on LP64 hosts; the dequantisation
// multiplies the int16 coefficient by the table entry narrowed to int16, as libjpeg's ISLOW_MULT_TYPE does, and the
// range-limit table: value + 128 clamped to 0..255 within +-512, libjpeg's wrap-around beyond.
constexpr int CONST_BITS = 13, PASS1_BITS = 2;

__device__ __forceinline__ void idct_1d(const long long *in, long long *o) {
  const long long z1e = (in[2] + in[6]) * 4433;             // FIX(0.541196100)
  const long long tmp2 = z1e - in[6] * 15137;                 // FIX(1.847759065)
  const long long tmp3 = z1e + in[2] * 6270;                  // FIX(0.765366865)
  const long long tmp0 = (in[0] + in[4]) * (1 << CONST_BITS);
  const long long tmp1 = (in[0] - in[4]) * (1 << CONST_BITS);
  const long long t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  long long a0 = in[7], a1 = in[5], a2 = in[3], a3 = in[1];
  long long z1 = a0 + a3, z2 = a1 + a2, z3 = a0 + a2, z4 = a1 + a3;
  const long long z5 = (z3 + z4) * 9633;                      // FIX(1.175875602)
  a0 *= 2446;                                           // FIX(0.298631336)
  a1 *= 16819;                                          // FIX(2.053119869)
  a2 *= 25172;                                          // FIX(3.072711026)
  a3 *= 12299;                                          // FIX(1.501321110)
  z1 *= -7373;                                          // -FIX(0.899976223)
  z2 *= -20995;                                         // -FIX(2.562915447)
  z3 = z3 * -16069 + z5;                                // -FIX(1.961570560)
  z4 = z4 * -3196 + z5;                                 // -FIX(0.390180644)
  a0 += z1 + z3;
  a1 += z2 + z4;
  a2 += z2 + z3;
  a3 += z1 + z4;
  o[0] = t10 + a3; o[7] = t10 - a3;
  o[1] = t11 + a2; o[6] = t11 - a2;
  o[2] = t12 + a1; o[5] = t12 - a1;
  o[3] = t13 + a0; o[4] = t13 - a0;
}

__device__ __forceinline__ unsigned range_limit(int v) {
  const int i = v & 1023;
  return i < 128 ? i + 128 : i < 512 ? 255 : i < 896 ? 0 : i - 896;
}

constexpr int IDCT_BLOCKS = 32;  // blocks per CTA, 8 threads each

__global__ void __launch_bounds__(IDCT_BLOCKS * 8) idct_kernel(const int16_t *__restrict__ coef, const int *__restrict__ quant,
                                                               Geom g, uint8_t *planes) {
  __shared__ int ws[IDCT_BLOCKS][8][9];
  pdl_prologue();
  const int lb = threadIdx.x >> 3, j = threadIdx.x & 7;
  const long long b = (long long)blockIdx.x * IDCT_BLOCKS + lb;
  const bool live = b < g.n_blocks;
  int comp = 0, by = 0, bx = 0;
  if (live) {
    if (g.ncomp == 1) {
      by = (int)(b / g.mx);
      bx = (int)(b - (long long)by * g.mx);
    } else {
      const long long mcu = b / g.bpm;
      const int w = (int)(b - mcu * g.bpm);
      comp = g.blk_comp[w];
      const int my_ = (int)(mcu / g.mx), mx_ = (int)(mcu - (long long)my_ * g.mx);
      by = my_ * g.comp_v[comp] + g.blk_dy[w];
      bx = mx_ * g.comp_h[comp] + g.blk_dx[w];
    }
    // pass 1: column j
    const int *q = quant + g.q_tab[comp] * 64;
    long long in[8], o[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) in[r] = (int)coef[b * 64 + r * 8 + j] * (int)(int16_t)__ldg(q + r * 8 + j);
    idct_1d(in, o);
#pragma unroll
    for (int r = 0; r < 8; ++r) ws[lb][r][j] = (int)((o[r] + (1 << (CONST_BITS - PASS1_BITS - 1))) >> (CONST_BITS - PASS1_BITS));
  }
  __syncthreads();
  if (!live) return;
  // pass 2: row j
  long long in[8], o[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) in[c] = ws[lb][j][c];
  idct_1d(in, o);
  unsigned lo = 0, hi = 0;
  constexpr int SH = CONST_BITS + PASS1_BITS + 3;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    lo |= range_limit((int)((o[c] + (1 << (SH - 1))) >> SH)) << (8 * c);
    hi |= range_limit((int)((o[c + 4] + (1 << (SH - 1))) >> SH)) << (8 * c);
  }
  uint8_t *dst = planes + g.plane_off[comp] + (long long)(by * 8 + j) * g.plane_w[comp] + bx * 8;
  *reinterpret_cast<uint2 *>(dst) = make_uint2(lo, hi);
}

// ---- upsampling + colour + orientation -------------------------------------------------------------------------------
// libjpeg "fancy" upsampling (used when the chroma row has more than 2 samples; plain replication otherwise):
//   h2v1: output 2i = (3 s[i] + s[i-1] + 1) >> 2, output 2i+1 = (3 s[i] + s[i+1] + 2) >> 2; the first and last outputs copy
//         the edge sample.
//   h2v2: per column first the vertical sum cs = 3 s[row] + s[row -+ 1] (the nearer chroma row for output rows 2j / 2j+1,
//         the edge row repeated above the top and below the last real row), then horizontally
//         output 2i = (3 cs[i] + cs[i-1] + 8) >> 4, 2i+1 = (3 cs[i] + cs[i+1] + 7) >> 4, edges (4 cs + 8) >> 4 / (4 cs + 7) >> 4.
__device__ __forceinline__ int chroma(const uint8_t *pl, int pw, const Geom &g, int y, int x) {
  if (g.hmax == 1) return pl[(long long)y * pw + x];
  const int i = x >> 1;
  const bool odd = x & 1;
  if (g.dw <= 2) return pl[(long long)(g.vmax == 2 ? y >> 1 : y) * pw + i];
  const int n = odd ? i + 1 : i - 1;
  const bool edge = odd ? i == g.dw - 1 : i == 0;
  if (g.vmax == 1) {
    const uint8_t *row = pl + (long long)y * pw;
    const int s = row[i];
    return edge ? s : (3 * s + row[n] + (odd ? 2 : 1)) >> 2;
  }
  const int j = y >> 1;
  const int jn = (y & 1) ? min(j + 1, g.dh - 1) : max(j - 1, 0);
  const uint8_t *r0 = pl + (long long)j * pw, *r1 = pl + (long long)jn * pw;
  const int cs = 3 * r0[i] + r1[i];
  if (edge) return (4 * cs + (odd ? 7 : 8)) >> 4;
  const int cn = 3 * r0[n] + r1[n];
  return (3 * cs + cn + (odd ? 7 : 8)) >> 4;
}

__global__ void __launch_bounds__(256) colour_kernel(const uint8_t *__restrict__ planes, Geom g, int out_h, int out_w,
                                                     uint8_t *__restrict__ out) {
  pdl_prologue();
  const int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
  if (c >= out_w) return;
  const int H = g.height, W = g.width;
  int y, x;  // source pixel of output (r, c): PIL's transpose for EXIF orientations 2..8
  switch (g.orientation) {
    case 2: y = r; x = W - 1 - c; break;
    case 3: y = H - 1 - r; x = W - 1 - c; break;
    case 4: y = H - 1 - r; x = c; break;
    case 5: y = c; x = r; break;
    case 6: y = H - 1 - c; x = r; break;
    case 7: y = H - 1 - c; x = W - 1 - r; break;
    case 8: y = c; x = W - 1 - r; break;
    default: y = r; x = c; break;
  }
  const int Y = planes[g.plane_off[0] + (long long)y * g.plane_w[0] + x];
  int R, G, B;
  if (g.ncomp == 1) {
    R = G = B = Y;
  } else {
    // libjpeg ycc_rgb_convert: FIX(x) = round(x * 2^16); R and B terms rounded per value, G rounded once after the sum
    const int cb = chroma(planes + g.plane_off[1], g.plane_w[1], g, y, x) - 128;
    const int cr = chroma(planes + g.plane_off[2], g.plane_w[2], g, y, x) - 128;
    R = min(max(Y + ((91881 * cr + 32768) >> 16), 0), 255);                // FIX(1.40200)
    G = min(max(Y + ((-22554 * cb - 46802 * cr + 32768) >> 16), 0), 255);  // FIX(0.34414), FIX(0.71414)
    B = min(max(Y + ((116130 * cb + 32768) >> 16), 0), 255);               // FIX(1.77200)
  }
  uint8_t *o = out + ((long long)r * out_w + c) * 3;
  o[0] = (uint8_t)(g.bgr ? B : R);
  o[1] = (uint8_t)G;
  o[2] = (uint8_t)(g.bgr ? R : B);
}

struct Layout {
  long long coef, planes, E, X0, A0, X1, A1, P, total;
};

int make_geom(Geom &g, int scan_bytes, const int *comp, int ncomp, int height, int width, int restart_interval, int orientation,
              int bgr) {
  if (scan_bytes <= 0 || height <= 0 || width <= 0 || (ncomp != 1 && ncomp != 3) || restart_interval < 0)
    return fail(APE_ERR_INVALID_ARG, "jpeg: bad geometry (scan %d bytes, %dx%d, %d components)", scan_bytes, height, width, ncomp);
  g = Geom{};
  g.ncomp = ncomp;
  g.width = width;
  g.height = height;
  g.scan_bytes = scan_bytes;
  g.orientation = orientation;
  g.bgr = bgr ? 1 : 0;
  g.restart_interval = restart_interval;
  for (int c = 0; c < ncomp; ++c) {
    g.comp_h[c] = ncomp == 1 ? 1 : comp[4 * c + 3] >> 4;
    g.comp_v[c] = ncomp == 1 ? 1 : comp[4 * c + 3] & 15;
    g.dc_tab[c] = comp[4 * c];
    g.ac_tab[c] = comp[4 * c + 1];
    g.q_tab[c] = comp[4 * c + 2];
    if (g.dc_tab[c] < 0 || g.dc_tab[c] >= MAX_TABLES || g.ac_tab[c] < 0 || g.ac_tab[c] >= MAX_TABLES || g.q_tab[c] < 0 || g.q_tab[c] > 3)
      return fail(APE_ERR_INVALID_ARG, "jpeg: table index out of range");
  }
  g.hmax = g.comp_h[0];
  g.vmax = g.comp_v[0];
  if (ncomp == 3) {
    const bool ok = (g.hmax == 1 && g.vmax == 1) || (g.hmax == 2 && g.vmax == 1) || (g.hmax == 2 && g.vmax == 2);
    if (!ok || g.comp_h[1] != 1 || g.comp_v[1] != 1 || g.comp_h[2] != 1 || g.comp_v[2] != 1)
      return fail(APE_ERR_UNSUPPORTED, "jpeg: sampling %dx%d over chroma %dx%d,%dx%d", g.hmax, g.vmax, g.comp_h[1], g.comp_v[1],
                  g.comp_h[2], g.comp_v[2]);
  }
  g.mx = (width + 8 * g.hmax - 1) / (8 * g.hmax);
  g.my = (height + 8 * g.vmax - 1) / (8 * g.vmax);
  g.dw = (width + g.hmax - 1) / g.hmax;
  g.dh = (height + g.vmax - 1) / g.vmax;
  int n = 0;
  for (int c = 0; c < ncomp; ++c)
    for (int dy = 0; dy < g.comp_v[c]; ++dy)
      for (int dx = 0; dx < g.comp_h[c]; ++dx) {
        g.blk_comp[n] = c;
        g.blk_dy[n] = dy;
        g.blk_dx[n] = dx;
        ++n;
      }
  g.bpm = n;
  g.n_blocks = g.mx * g.my * g.bpm;
  long long off = 0;
  for (int c = 0; c < ncomp; ++c) {
    g.plane_w[c] = g.mx * g.comp_h[c] * 8;
    g.plane_h[c] = g.my * g.comp_v[c] * 8;
    g.plane_off[c] = off;
    off += (long long)g.plane_w[c] * g.plane_h[c];
  }
  g.n_sub = (scan_bytes + SUBSEQ_BYTES - 1) / SUBSEQ_BYTES;
  g.n_intervals = restart_interval ? (g.mx * g.my + restart_interval - 1) / restart_interval : 0;
  return APE_OK;
}

Layout make_layout(const Geom &g) {
  auto up = [](long long x) { return (x + 255) & ~255ll; };
  Layout L;
  long long o = 0;
  L.coef = o; o += up((long long)g.n_blocks * 128);
  L.planes = o;
  long long pb = 0;
  for (int c = 0; c < g.ncomp; ++c) pb += (long long)g.plane_w[c] * g.plane_h[c];
  o += up(pb);
  const long long s = up((long long)g.n_sub * 16);
  L.E = o; o += s;
  L.X0 = o; o += s;
  L.A0 = o; o += s;
  L.X1 = o; o += s;
  L.A1 = o; o += s;
  L.P = o; o += s;
  L.total = o;
  return L;
}

}  // namespace
}  // namespace ape

extern "C" int64_t ape_jpeg_workspace_bytes(int scan_bytes, const int *comp, int ncomp, int height, int width, int restart_interval) {
  using namespace ape;
  Geom g;
  if (make_geom(g, scan_bytes, comp, ncomp, height, width, restart_interval, 1, 0) != APE_OK) return -1;
  return make_layout(g).total;
}

extern "C" int ape_jpeg_decode(const uint8_t *scan, int scan_bytes, const int *huff, int n_tables, const int *quant,
                               const int *comp, int ncomp, int height, int width, int restart_interval, const int *restart_offsets,
                               int orientation, int bgr, void *workspace, int64_t workspace_bytes, int *status, uint8_t *out,
                               void *stream) {
  using namespace ape;
  if (!scan || !huff || !quant || !comp || !workspace || !status || !out) return fail(APE_ERR_NULL_PTR, "jpeg: null pointer");
  if (n_tables < 1 || n_tables > MAX_TABLES) return fail(APE_ERR_INVALID_ARG, "jpeg: %d Huffman tables", n_tables);
  Geom g;
  int rc = make_geom(g, scan_bytes, comp, ncomp, height, width, restart_interval, orientation, bgr);
  if (rc) return rc;
  if (g.n_intervals > 1 && !restart_offsets) return fail(APE_ERR_NULL_PTR, "jpeg: restart offsets missing");
  const Layout L = make_layout(g);
  if (workspace_bytes < L.total) return fail(APE_ERR_INVALID_ARG, "jpeg: workspace of %lld bytes, %lld needed",
                                             (long long)workspace_bytes, (long long)L.total);
  cudaStream_t st = (cudaStream_t)stream;
  char *ws = (char *)workspace;
  int16_t *coef = (int16_t *)(ws + L.coef);
  uint8_t *planes = (uint8_t *)(ws + L.planes);
  int4 *E = (int4 *)(ws + L.E), *X0 = (int4 *)(ws + L.X0), *A0 = (int4 *)(ws + L.A0), *X1 = (int4 *)(ws + L.X1),
       *A1 = (int4 *)(ws + L.A1), *P = (int4 *)(ws + L.P);
  const size_t smem = (size_t)n_tables * TABLE_WORDS * sizeof(int);
  if (cudaMemsetAsync(status, 0, sizeof(int), st) != cudaSuccess || cudaMemsetAsync(coef, 0, (size_t)g.n_blocks * 128, st) != cudaSuccess)
    return check_launch("jpeg: memset");
  if (g.restart_interval) {
    const int grid = (g.n_intervals + DEC_THREADS - 1) / DEC_THREADS;
    APE_LAUNCH(huff_write_kernel, grid, DEC_THREADS, smem, st, scan, huff, n_tables, g, (const int4 *)nullptr,
               (const int4 *)nullptr, 1, restart_offsets, coef, status);
    if ((rc = check_launch("jpeg huff_write_kernel"))) return rc;
  } else {
    const int grid = (g.n_sub + DEC_THREADS - 1) / DEC_THREADS;
    APE_LAUNCH(huff_spec_kernel, grid, DEC_THREADS, smem, st, scan, huff, n_tables, g, E, X0, A0);
    if ((rc = check_launch("jpeg huff_spec_kernel"))) return rc;
    APE_LAUNCH(huff_prop_kernel, grid, DEC_THREADS, smem, st, scan, huff, n_tables, g, E, (const int4 *)X0, (const int4 *)A0, X1, A1);
    if ((rc = check_launch("jpeg huff_prop_kernel"))) return rc;
    APE_LAUNCH(huff_chain_kernel, 1, 32, smem, st, scan, huff, n_tables, g, E, (const int4 *)X1, (const int4 *)A1, P, status);
    if ((rc = check_launch("jpeg huff_chain_kernel"))) return rc;
    APE_LAUNCH(huff_write_kernel, grid, DEC_THREADS, smem, st, scan, huff, n_tables, g, (const int4 *)E, (const int4 *)P,
               0, (const int *)nullptr, coef, status);
    if ((rc = check_launch("jpeg huff_write_kernel"))) return rc;
  }
  APE_LAUNCH(idct_kernel, (unsigned)((g.n_blocks + IDCT_BLOCKS - 1) / IDCT_BLOCKS), IDCT_BLOCKS * 8, 0, st, coef, quant, g, planes);
  if ((rc = check_launch("jpeg idct_kernel"))) return rc;
  const bool swap = orientation >= 5 && orientation <= 8;
  const int out_h = swap ? width : height, out_w = swap ? height : width;
  APE_LAUNCH(colour_kernel, dim3((out_w + 255) / 256, out_h), 256, 0, st, (const uint8_t *)planes, g, out_h, out_w, out);
  return check_launch("jpeg colour_kernel");
}

extern "C" int ape_jpeg_status_error(int status) {
  using namespace ape;
  if (status == 0) return APE_OK;
  return fail(APE_ERR_INVALID_ARG, "jpeg: corrupt scan:%s%s%s", (status & ERR_BAD_CODE) ? " invalid Huffman code" : "",
              (status & ERR_TRUNCATED) ? " data ends inside a needed codeword" : "",
              (status & ERR_SHORT) ? " fewer blocks than the frame holds" : "");
}
