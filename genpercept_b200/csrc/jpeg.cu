// Baseline JPEG decoding on the GPU, byte for byte as Pillow (libjpeg-turbo, JDCT_ISLOW, fancy upsampling) decodes it.
//
//   host:   marker parser, canonical Huffman tables, acceptance (gp_jpeg_probe); workspace layout
//   device: find the scan's terminating marker -> unstuff (drop the 0x00 after 0xFF, remove RSTn and record where each
//           restart interval starts) with a block-wide scan -> cut each interval into subsequences of kSubBits bits ->
//           self-synchronising Huffman passes (Weissenberger & Schmidt, "Massively Parallel Huffman Decoding on
//           GPUs", ICPP 2018): each subsequence decodes from its entry state (bit, block of the MCU, coefficient) to
//           its end, and its exit becomes the next entry, until no entry changes -> a segmented scan of the block
//           counts and DC differences per interval -> the writing pass -> ISLOW IDCT per block -> upsampling and
//           YCbCr -> RGB into the caller's strided uint8 output.
// Everything the device derives from stream content is bounded; a violation sets a status bit and the call returns
// GP_ERR_INVALID (as does a decode that did not converge within kMaxPasses), so the caller can take Pillow's path.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <string>

#include "status.h"

namespace {

constexpr int kSubBits = 4096;      // subsequence length; oracle/jpeg.py's simulate_sync needs 3 passes on the fixtures
constexpr int kMaxPasses = 1024;    // past this the decode reports "not converged"
constexpr int kPassBatch = 4;       // passes launched between two reads of the convergence flag
constexpr int kChunk = 4096;        // bytes of the entropy-coded segment per unstuffing CTA (256 threads x 16)
constexpr int kScan = 1024;         // elements per scan CTA

enum : int {
  ST_MARKER = 1,       // no EOI after the scan, or another marker inside it
  ST_RESTART = 2,      // restart markers out of sequence or not one per interval
  ST_HUFFMAN = 4,      // invalid code or a run past coefficient 63 in a block of the frame
  ST_EXHAUSTED = 8,    // an interval's data ended before its last block
  ST_CONVERGE = 16,    // the synchronisation passes did not converge
  ST_COUNT = 32,       // the number of decoded blocks differs from the frame's
  ST_DC = 64,          // an absolute DC value outside int16
  ST_LAYOUT = 128,     // more subsequences than the workspace holds
  ST_RANGE = 256       // an IDCT value outside the range where libjpeg-turbo's C and SIMD IDCTs agree
};

const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                             41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                             30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct HuffDev {                    // libjpeg's d_derived_tbl, restated: a 9-bit lookup and the per-length bounds
  uint16_t fast[512];               // (length << 8) | symbol for codes of <= 9 bits; 0 = longer or invalid
  int32_t maxcode[17];              // largest code of each length, -1 if none
  int32_t valoff[17];               // index into vals of a code of that length = valoff + code
  uint8_t vals[256];
};

struct Tables {                     // uploaded with the file bytes
  HuffDev dc[4], ac[4];
  uint16_t qt[4][64];               // natural order
};

struct Geo {                        // everything else the kernels need, passed by value
  int W, H, mcus_x, mcus_y, bpm, ri, n_int, hY, vY;
  int blk_comp[6], blk_dy[6], blk_dx[6];
  int td[3], ta[3], tq[3], bw[3], bh[3];
  long long coef_off[3], pix_off[3];      // per component, in elements of the coefficient / pixel regions
  uint8_t zz[64];
};

struct Header {
  int W = 0, H = 0, dri = 0;
  long long start = 0;              // first byte of the entropy-coded segment
  int id[3], h[3], v[3], tq[3], td[3], ta[3];
  bool has_qt[4] = {}, has_dc[4] = {}, has_ac[4] = {};
  Tables t;
};

struct S4 { long long v[4]; };

struct State {                      // device-side status block
  int status;
  int end;                          // offset of the terminating marker in the entropy-coded segment
  unsigned long long blocks_done;
  long long n_sub;
  int changed[kMaxPasses];
};

// ------------------------------------------------------------------------------------------------ host parser
[[noreturn]] void reject(const char* why) { throw gp::GpError(GP_ERR_INVALID, why); }

void build_huff(const uint8_t* counts, const uint8_t* vals, int n, bool dc, HuffDev& t) {
  memset(&t, 0, sizeof t);
  for (int i = 0; i < n; ++i) {
    if (dc && vals[i] > 15) reject("bad DC Huffman table");
    t.vals[i] = vals[i];
  }
  int code = 0, k = 0;
  for (int len = 1; len <= 16; ++len) {
    const int c = counts[len - 1];
    t.valoff[len] = k - code;
    t.maxcode[len] = c ? code + c - 1 : -1;
    for (int j = 0; j < c; ++j, ++code, ++k)
      if (len <= 9)
        for (int f = code << (9 - len); f < (code + 1) << (9 - len); ++f) t.fast[f] = (uint16_t)(len << 8 | vals[k]);
    if (code >= (1 << len)) reject("bad Huffman table");   // libjpeg: the all-ones code of a length is reserved
    code <<= 1;
  }
}

Header parse(const uint8_t* d, size_t n) {
  Header hd;
  if (!d || n < 4 || d[0] != 0xFF || d[1] != 0xD8) reject("no SOI");
  size_t i = 2;
  bool jfif = false, frame = false;
  int adobe = -1;
  for (;;) {
    if (i + 4 > n) reject("truncated header");
    if (d[i] != 0xFF) reject("expected a marker");
    const int m = d[i + 1];
    if (m == 0xFF) { ++i; continue; }
    const size_t L = (size_t)d[i + 2] << 8 | d[i + 3];
    if (L < 2 || i + 2 + L > n) reject("bad segment length");
    const uint8_t* seg = d + i + 4;
    const size_t sl = L - 2;
    if (m == 0xE0 && sl >= 14 && !memcmp(seg, "JFIF\0", 5)) {
      jfif = true;
    } else if (m == 0xEE && sl >= 12 && !memcmp(seg, "Adobe", 5)) {
      adobe = seg[11];
    } else if (m == 0xDB) {
      for (size_t j = 0; j < sl;) {
        const int pq = seg[j] >> 4, tq = seg[j] & 15;
        const size_t nb = pq ? 128 : 64;
        if (pq > 1 || tq > 3 || j + 1 + nb > sl) reject("bad DQT");
        for (int z = 0; z < 64; ++z)
          hd.t.qt[tq][kZigzag[z]] = pq ? (uint16_t)(seg[j + 1 + 2 * z] << 8 | seg[j + 2 + 2 * z]) : seg[j + 1 + z];
        hd.has_qt[tq] = true;
        j += 1 + nb;
      }
    } else if (m == 0xC4) {
      for (size_t j = 0; j < sl;) {
        if (j + 17 > sl) reject("bad DHT");
        const int tc = seg[j] >> 4, th = seg[j] & 15;
        int cnt = 0;
        for (int l = 0; l < 16; ++l) cnt += seg[j + 1 + l];
        if (tc > 1 || th > 3 || cnt > 256 || j + 17 + cnt > sl) reject("bad DHT");
        build_huff(seg + j + 1, seg + j + 17, cnt, tc == 0, tc ? hd.t.ac[th] : hd.t.dc[th]);
        (tc ? hd.has_ac : hd.has_dc)[th] = true;
        j += 17 + cnt;
      }
    } else if (m == 0xDD) {
      if (L != 4) reject("bad DRI");
      hd.dri = seg[0] << 8 | seg[1];
    } else if (m == 0xC0 || m == 0xC1) {
      if (frame || sl < 6) reject("bad SOF");
      if (seg[0] != 8 || seg[5] != 3 || sl != 15) reject("not 8-bit, 3-component");
      hd.H = seg[1] << 8 | seg[2];
      hd.W = seg[3] << 8 | seg[4];
      if (!hd.H || !hd.W) reject("zero-sized frame");
      for (int c = 0; c < 3; ++c) {
        hd.id[c] = seg[6 + 3 * c];
        hd.h[c] = seg[7 + 3 * c] >> 4;
        hd.v[c] = seg[7 + 3 * c] & 15;
        hd.tq[c] = seg[8 + 3 * c];
      }
      frame = true;
    } else if (m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
      reject("not a sequential Huffman frame");
    } else if (m == 0xDA) {
      if (!frame) reject("SOS before SOF");
      if (sl < 1 || seg[0] != 3 || sl != 10) reject("not one interleaved scan of all components");
      for (int c = 0; c < 3; ++c) {
        if (seg[1 + 2 * c] != hd.id[c]) reject("scan component order");
        hd.td[c] = seg[2 + 2 * c] >> 4;
        hd.ta[c] = seg[2 + 2 * c] & 15;
      }
      if (seg[7] != 0 || seg[8] != 63 || seg[9] != 0) reject("not a sequential scan");
      hd.start = (long long)(i + 2 + L);
      break;
    } else if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7)) {
      reject("unexpected marker");
    }
    i += 2 + L;
  }
  // libjpeg's default_decompress_parms for 3 components: JFIF, else Adobe's transform, else the component ids
  if (!jfif) {
    if (adobe >= 0) {
      if (adobe != 1) reject("Adobe transform is not YCbCr");
    } else if (hd.id[0] != 1 || hd.id[1] != 2 || hd.id[2] != 3) {
      reject("colour space not inferred as YCbCr");
    }
  }
  const bool luma_ok =
      (hd.h[0] == 1 && hd.v[0] == 1) || (hd.h[0] == 2 && hd.v[0] == 1) || (hd.h[0] == 2 && hd.v[0] == 2);
  if (!luma_ok || hd.h[1] != 1 || hd.v[1] != 1 || hd.h[2] != 1 || hd.v[2] != 1) reject("sampling");
  for (int c = 0; c < 3; ++c)
    if (hd.tq[c] > 3 || !hd.has_qt[hd.tq[c]] || hd.td[c] > 3 || !hd.has_dc[hd.td[c]] || hd.ta[c] > 3 ||
        !hd.has_ac[hd.ta[c]])
      reject("missing table");
  return hd;
}

// ------------------------------------------------------------------------------------------------ workspace layout
struct Layout {
  Geo g;
  long long L, n_chunks, n_sub_max, n_blocks, coef_elems, pix_bytes;
  size_t o_file, o_tab, o_state, o_chunk, o_chunk_f, o_chunk_b, o_chunk_bf, o_u, o_rst, o_iv, o_iv_f, o_iv_b,
      o_iv_bf, o_iv_se, o_sub, o_e0, o_e1, o_used, o_exit, o_agg, o_agg_f, o_agg_b, o_agg_bf, o_coef, o_pix, total;
};

size_t carve(size_t& at, size_t bytes) {
  const size_t o = at;
  at += (bytes + 255) / 256 * 256;
  return o;
}

Layout plan(const Header& hd, size_t nbytes) {
  Layout y;
  Geo& g = y.g;
  memset(&g, 0, sizeof g);
  g.W = hd.W;
  g.H = hd.H;
  g.hY = hd.h[0];
  g.vY = hd.v[0];
  g.mcus_x = (hd.W + 8 * g.hY - 1) / (8 * g.hY);
  g.mcus_y = (hd.H + 8 * g.vY - 1) / (8 * g.vY);
  const long long total_mcus = (long long)g.mcus_x * g.mcus_y;
  g.ri = hd.dri ? hd.dri : (int)total_mcus;
  g.n_int = (int)((total_mcus + g.ri - 1) / g.ri);
  int b = 0;
  for (int c = 0; c < 3; ++c)
    for (int dy = 0; dy < hd.v[c]; ++dy)
      for (int dx = 0; dx < hd.h[c]; ++dx, ++b) {
        g.blk_comp[b] = c;
        g.blk_dy[b] = dy;
        g.blk_dx[b] = dx;
      }
  g.bpm = b;
  long long coef = 0, pix = 0;
  for (int c = 0; c < 3; ++c) {
    g.td[c] = hd.td[c];
    g.ta[c] = hd.ta[c];
    g.tq[c] = hd.tq[c];
    g.bw[c] = g.mcus_x * hd.h[c];
    g.bh[c] = g.mcus_y * hd.v[c];
    g.coef_off[c] = coef;
    g.pix_off[c] = pix;
    coef += (long long)g.bw[c] * g.bh[c] * 64;
    pix += (long long)g.bw[c] * g.bh[c] * 64;
  }
  memcpy(g.zz, kZigzag, 64);
  y.n_blocks = coef / 64;
  y.coef_elems = coef;
  y.pix_bytes = pix;
  y.L = (long long)nbytes - hd.start;
  if (y.L < 2) reject("no entropy-coded data");
  if (y.L >= (1LL << 28)) reject("entropy-coded segment above 256 MiB");
  y.n_chunks = (y.L + kChunk - 1) / kChunk;
  y.n_sub_max = g.n_int + (8 * y.L + kSubBits - 1) / kSubBits + 1;
  auto nb = [](long long n) { return (n + kScan - 1) / kScan; };
  size_t at = 0;
  y.o_file = carve(at, nbytes);
  y.o_tab = carve(at, sizeof(Tables));
  y.o_state = carve(at, sizeof(State));
  y.o_chunk = carve(at, y.n_chunks * sizeof(S4));
  y.o_chunk_f = carve(at, y.n_chunks);
  y.o_chunk_b = carve(at, nb(y.n_chunks) * sizeof(S4));
  y.o_chunk_bf = carve(at, nb(y.n_chunks));
  y.o_u = carve(at, y.L + 16);
  y.o_rst = carve(at, (size_t)g.n_int * 4);
  y.o_iv = carve(at, (size_t)g.n_int * sizeof(S4));
  y.o_iv_f = carve(at, g.n_int);
  y.o_iv_b = carve(at, nb(g.n_int) * sizeof(S4));
  y.o_iv_bf = carve(at, nb(g.n_int));
  y.o_iv_se = carve(at, (size_t)g.n_int * 8);
  y.o_sub = carve(at, y.n_sub_max * 16);
  y.o_e0 = carve(at, y.n_sub_max * 8);
  y.o_e1 = carve(at, y.n_sub_max * 8);
  y.o_used = carve(at, y.n_sub_max * 8);
  y.o_exit = carve(at, y.n_sub_max * 8);
  y.o_agg = carve(at, y.n_sub_max * sizeof(S4));
  y.o_agg_f = carve(at, y.n_sub_max);
  y.o_agg_b = carve(at, nb(y.n_sub_max) * sizeof(S4));
  y.o_agg_bf = carve(at, nb(y.n_sub_max));
  y.o_coef = carve(at, coef * 2);
  y.o_pix = carve(at, pix);
  y.total = at;
  return y;
}

// ------------------------------------------------------------------------------------------------ device: scans
// Inclusive segmented scan of S4 sums (a head flag restarts the sum), in place, over three kernels.
__device__ __forceinline__ void seg_combine(S4& acc, uint8_t& af, const S4& prev, uint8_t pf) {
  if (!af)
    for (int j = 0; j < 4; ++j) acc.v[j] += prev.v[j];
  af |= pf;
}

__device__ void block_scan(S4& x, uint8_t& f, S4* sh, uint8_t* shf) {
  const int t = threadIdx.x;
  sh[t] = x;
  shf[t] = f;
  __syncthreads();
  for (int off = 1; off < blockDim.x; off <<= 1) {
    S4 p;
    uint8_t pf = 0;
    const bool has = t >= off;
    if (has) {
      p = sh[t - off];
      pf = shf[t - off];
    }
    __syncthreads();
    if (has) seg_combine(x, f, p, pf);
    sh[t] = x;
    shf[t] = f;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kScan) scan_local(S4* x, uint8_t* flag, long long n, S4* bagg, uint8_t* bflag) {
  __shared__ S4 sh[kScan];
  __shared__ uint8_t shf[kScan];
  const long long i = (long long)blockIdx.x * kScan + threadIdx.x;
  S4 v = {};
  uint8_t f = 0;
  if (i < n) {
    v = x[i];
    f = flag[i];
  }
  block_scan(v, f, sh, shf);
  if (i < n) {
    x[i] = v;
    flag[i] = f;
  }
  if (threadIdx.x == kScan - 1) {
    bagg[blockIdx.x] = v;
    bflag[blockIdx.x] = f;
  }
}

__global__ void __launch_bounds__(kScan) scan_top(S4* bagg, uint8_t* bflag, long long nb) {
  __shared__ S4 sh[kScan];
  __shared__ uint8_t shf[kScan];
  __shared__ S4 carry;
  __shared__ uint8_t carryf;
  if (threadIdx.x == 0) {
    carry = S4{};
    carryf = 0;
  }
  __syncthreads();
  for (long long base = 0; base < nb; base += kScan) {
    const long long i = base + threadIdx.x;
    S4 v = {};
    uint8_t f = 0;
    if (i < nb) {
      v = bagg[i];
      f = bflag[i];
    }
    block_scan(v, f, sh, shf);
    seg_combine(v, f, carry, carryf);
    if (i < nb) {
      bagg[i] = v;
      bflag[i] = f;
    }
    __syncthreads();
    if (threadIdx.x == kScan - 1) {
      carry = v;
      carryf = f;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kScan) scan_add(S4* x, const uint8_t* flag, long long n, const S4* bagg) {
  const long long i = (long long)blockIdx.x * kScan + threadIdx.x;
  if (i >= n || blockIdx.x == 0 || flag[i]) return;
  const S4 c = bagg[blockIdx.x - 1];
  for (int j = 0; j < 4; ++j) x[i].v[j] += c.v[j];
}

void scan(S4* x, uint8_t* flag, long long n, S4* bagg, uint8_t* bflag, cudaStream_t s) {
  const long long nb = (n + kScan - 1) / kScan;
  scan_local<<<(unsigned)nb, kScan, 0, s>>>(x, flag, n, bagg, bflag);
  if (nb > 1) {
    scan_top<<<1, kScan, 0, s>>>(bagg, bflag, nb);
    scan_add<<<(unsigned)nb, kScan, 0, s>>>(x, flag, n, bagg);
  }
}

// ------------------------------------------------------------------------------------------------ device: unstuffing
__global__ void find_end(const uint8_t* E, long long L, State* st) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < L; i += (long long)gridDim.x * blockDim.x) {
    if (E[i] != 0xFF) continue;
    const int nx = i + 1 < L ? E[i + 1] : 0x100;
    if (!(nx == 0 || (nx >= 0xD0 && nx <= 0xD7))) atomicMin(&st->end, (int)i);
  }
}

// byte i (< end) of the segment: kept as data, and whether it starts a restart marker
__device__ __forceinline__ void classify(const uint8_t* E, long long i, bool& keep, bool& rst) {
  rst = false;
  if (i > 0 && E[i - 1] == 0xFF) {         // the stuffed 0x00 or a marker's second byte
    keep = false;
  } else if (E[i] == 0xFF) {
    keep = E[i + 1] == 0;
    rst = !keep;
  } else {
    keep = true;
  }
}

__global__ void __launch_bounds__(256) unstuff_count(const uint8_t* E, long long L, State* st, S4* chunks,
                                                     uint8_t* flags) {
  __shared__ int kept, rsts;
  if (threadIdx.x == 0) {
    kept = rsts = 0;
    if (blockIdx.x == 0) {
      const long long e = st->end;
      if (e >= L - 1 || E[e + 1] != 0xD9) atomicOr(&st->status, ST_MARKER);
    }
  }
  __syncthreads();
  const long long end = st->end;
  const long long i0 = (long long)blockIdx.x * kChunk + threadIdx.x * 16;
  int k = 0, r = 0;
  for (int j = 0; j < 16; ++j) {
    const long long i = i0 + j;
    if (i >= end) break;
    bool keep, rst;
    classify(E, i, keep, rst);
    k += keep;
    r += rst;
  }
  atomicAdd(&kept, k);
  atomicAdd(&rsts, r);
  __syncthreads();
  if (threadIdx.x == 0) {
    chunks[blockIdx.x] = S4{{kept, rsts, 0, 0}};
    flags[blockIdx.x] = 0;
  }
}

__global__ void __launch_bounds__(256) unstuff_write(const uint8_t* E, State* st, const S4* chunks, uint8_t* U,
                                                     uint32_t* rst_pos, int n_rst_max) {
  __shared__ int sk[256], sr[256];
  const long long end = st->end;
  const long long i0 = (long long)blockIdx.x * kChunk + threadIdx.x * 16;
  int k = 0, r = 0;
  for (int j = 0; j < 16; ++j) {
    const long long i = i0 + j;
    if (i >= end) break;
    bool keep, rst;
    classify(E, i, keep, rst);
    k += keep;
    r += rst;
  }
  sk[threadIdx.x] = k;
  sr[threadIdx.x] = r;
  __syncthreads();
  for (int off = 1; off < 256; off <<= 1) {
    const int a = threadIdx.x >= off ? sk[threadIdx.x - off] : 0, b = threadIdx.x >= off ? sr[threadIdx.x - off] : 0;
    __syncthreads();
    sk[threadIdx.x] += a;
    sr[threadIdx.x] += b;
    __syncthreads();
  }
  long long ko = blockIdx.x ? chunks[blockIdx.x - 1].v[0] : 0;       // chunks: inclusive sums
  long long ro = blockIdx.x ? chunks[blockIdx.x - 1].v[1] : 0;
  ko += sk[threadIdx.x] - k;
  ro += sr[threadIdx.x] - r;
  for (int j = 0; j < 16; ++j) {
    const long long i = i0 + j;
    if (i >= end) break;
    bool keep, rst;
    classify(E, i, keep, rst);
    if (keep) U[ko++] = E[i];
    if (rst) {
      if (ro >= n_rst_max || E[i + 1] - 0xD0 != (int)(ro & 7)) atomicOr(&st->status, ST_RESTART);
      else rst_pos[ro] = (uint32_t)ko;
      ++ro;
    }
  }
}

// interval i: bit range and subsequence count
__global__ void intervals(State* st, const S4* chunks, long long n_chunks, const uint32_t* rst_pos, int n_int,
                          S4* iv, uint8_t* ivf, uint2* iv_se) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_int) return;
  const S4 tot = chunks[n_chunks - 1];
  if (i == 0 && tot.v[1] != n_int - 1) atomicOr(&st->status, ST_RESTART);
  const uint32_t total_bits = (uint32_t)(tot.v[0] * 8);
  uint32_t a = i == 0 ? 0 : rst_pos[i - 1] * 8u, z = i == n_int - 1 ? total_bits : rst_pos[i] * 8u;
  if (a > total_bits) a = total_bits;       // only reachable with ST_RESTART set: keep the layout bounded
  if (z > total_bits) z = total_bits;
  if (z < a) z = a;
  const long long nsub = z > a ? ((long long)(z - a) + kSubBits - 1) / kSubBits : 1;
  iv[i] = S4{{nsub, 0, 0, 0}};
  ivf[i] = 0;
  iv_se[i] = make_uint2(a, z);
}

struct Sub { uint32_t a, z, iv, head; };

__device__ __forceinline__ unsigned long long pack(uint32_t p, int b, int k) {
  return (unsigned long long)p << 16 | (unsigned)b << 8 | (unsigned)k;
}
constexpr unsigned long long kDead = ~0ULL;
constexpr unsigned long long kUnused = ~1ULL;     // no packed state has its top 16 bits set

__global__ void subsequences(State* st, const S4* iv, const uint2* iv_se, int n_int, long long n_sub_max, Sub* subs,
                             unsigned long long* e0, unsigned long long* e1, unsigned long long* used,
                             uint8_t* aggf) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = iv[n_int - 1].v[0];
  if (s == 0) {
    if (total > n_sub_max) atomicOr(&st->status, ST_LAYOUT);
    st->n_sub = min(total, n_sub_max);
  }
  if (s >= total || s >= n_sub_max) return;
  int lo = 0, hi = n_int - 1;              // first interval whose inclusive count exceeds s
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (iv[mid].v[0] > s) hi = mid; else lo = mid + 1;
  }
  const long long first = iv[lo].v[0] - (lo ? iv[lo].v[0] - iv[lo - 1].v[0] : iv[0].v[0]);
  const uint2 se = iv_se[lo];
  const uint32_t a = se.x + (uint32_t)(s - first) * kSubBits;
  const uint32_t z = min(a + (uint32_t)kSubBits, se.y);
  subs[s] = Sub{a, z, (uint32_t)lo, s == first ? 1u : 0u};
  e0[s] = e1[s] = pack(a, 0, 0);
  used[s] = kUnused;
  aggf[s] = s == first;
}

// ------------------------------------------------------------------------------------------------ device: Huffman
__device__ __forceinline__ uint32_t peek32(const uint8_t* U, uint32_t p) {
  const uint8_t* q = U + (p >> 3);
  const uint32_t w = (uint32_t)q[0] << 24 | (uint32_t)q[1] << 16 | (uint32_t)q[2] << 8 | q[3];
  const int sh = p & 7;
  return sh ? (w << sh | q[4] >> (8 - sh)) : w;
}

// one codeword at w (MSB first) -> (length, symbol), length 0 = invalid
__device__ __forceinline__ int huff(const HuffDev& t, uint32_t w, int& sym) {
  const int f = t.fast[w >> 23];
  if (f) {
    sym = f & 255;
    return f >> 8;
  }
  for (int len = 10; len <= 16; ++len) {
    const int code = (int)(w >> (32 - len));
    if (code <= t.maxcode[len]) {
      const int idx = t.valoff[len] + code;
      if (idx < 0 || idx > 255) return 0;
      sym = t.vals[idx];
      return len;
    }
  }
  return 0;
}

__device__ __forceinline__ int extend(uint32_t bits, int s) {
  return bits < (1u << (s - 1)) ? (int)bits - (1 << s) + 1 : (int)bits;
}


// Decodes one subsequence from `entry` to the first codeword boundary at or past its end.  WRITE = false: returns the
// exit and accumulates the blocks started and the DC differences per component into acc.  WRITE = true: `carry`
// holds the blocks started and DC sums of the interval before this subsequence; the coefficients of the frame's
// blocks (index < expected within the interval) are written with DC made absolute, and any fault in them is reported.
template <bool WRITE>
__device__ unsigned long long run_sub(const Tables& T, const Geo& g, const uint8_t* U, uint32_t end,
                                      unsigned long long entry, S4& acc, const S4& carry, long long expected,
                                      long long mcu0, uint32_t iv_end, int16_t* coef, State* st) {
  if (entry == kDead) return kDead;
  uint32_t p = (uint32_t)(entry >> 16);
  int b = (int)(entry >> 8 & 255), k = (int)(entry & 255);
  if (b >= g.bpm || k >= 64) return kDead;
  long long idx = carry.v[0] - 1;          // the block being decoded: the last one started before this subsequence
  long long dc[3] = {carry.v[1], carry.v[2], carry.v[3]};
  int16_t* blk = nullptr;
  bool real = false;
  while (p < end) {
    const int c = g.blk_comp[b];
    if (k == 0) {
      ++idx;
      real = WRITE && idx >= 0 && idx < expected;
      if (real) {
        const long long m = mcu0 + idx / g.bpm;
        if (idx % g.bpm != b) {
          atomicOr(&st->status, ST_HUFFMAN);
          return kDead;
        }
        const long long row = (m / g.mcus_x) * (c ? 1 : g.vY) + g.blk_dy[b];
        const long long col = (m % g.mcus_x) * (c ? 1 : g.hY) + g.blk_dx[b];
        blk = coef + g.coef_off[c] + (row * g.bw[c] + col) * 64;
      }
    } else if (WRITE && idx == carry.v[0] - 1 && blk == nullptr) {   // entered mid-block
      real = idx >= 0 && idx < expected;
      if (real) {
        const long long m = mcu0 + idx / g.bpm;
        if (idx % g.bpm != b) {
          atomicOr(&st->status, ST_HUFFMAN);
          return kDead;
        }
        const long long row = (m / g.mcus_x) * (c ? 1 : g.vY) + g.blk_dy[b];
        const long long col = (m % g.mcus_x) * (c ? 1 : g.hY) + g.blk_dx[b];
        blk = coef + g.coef_off[c] + (row * g.bw[c] + col) * 64;
      }
    }
    const uint32_t w = peek32(U, p);
    int sym = 0;
    const int len = huff(k == 0 ? T.dc[g.td[c]] : T.ac[g.ta[c]], w, sym);
    if (!len) {
      if (real) atomicOr(&st->status, ST_HUFFMAN);
      return kDead;
    }
    const uint32_t xw = w << len;
    if (k == 0) {
      const int v = sym ? extend(xw >> (32 - sym), sym) : 0;
      p += len + sym;
      if (!WRITE) {
        acc.v[0] += 1;
        acc.v[1 + c] += v;
      } else if (real) {
        dc[c] += v;
        if (dc[c] < -32768 || dc[c] > 32767) atomicOr(&st->status, ST_DC);
        blk[0] = (int16_t)dc[c];
      }
      k = 1;
    } else {
      const int r = sym >> 4, s = sym & 15;
      if (s) {
        k += r;
        if (k > 63) {
          if (real) atomicOr(&st->status, ST_HUFFMAN);
          return kDead;
        }
        if (real) blk[g.zz[k]] = (int16_t)extend(xw >> (32 - s), s);
        p += len + s;
        ++k;
      } else if (r == 15) {
        k += 16;
        p += len;
        if (k > 64) {
          if (real) atomicOr(&st->status, ST_HUFFMAN);
          return kDead;
        }
      } else {
        p += len;
        k = 64;
      }
    }
    // a block of the frame may not read past its interval's data (libjpeg would substitute zeros there)
    if (real && p > iv_end) atomicOr(&st->status, ST_EXHAUSTED);
    if (k == 64) {
      if (real) atomicAdd(&st->blocks_done, 1ULL);
      k = 0;
      blk = nullptr;
      real = false;
      if (++b == g.bpm) b = 0;
    }
  }
  return pack(p, b, k);
}

__device__ void load_huff(Tables& T, const Tables* tab) {
  constexpr int n = (int)(sizeof(HuffDev) * 8 / 4);
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    reinterpret_cast<uint32_t*>(&T)[i] = reinterpret_cast<const uint32_t*>(tab)[i];
  __syncthreads();
}

__global__ void __launch_bounds__(128) sync_pass(const Tables* tab, Geo g, const uint8_t* U, const Sub* subs,
                                                 State* st, int pass, const unsigned long long* ecur,
                                                 unsigned long long* enext, unsigned long long* used,
                                                 unsigned long long* exits, S4* agg) {
  if (pass > 0 && st->changed[pass - 1] == 0) return;      // converged in an earlier pass
  __shared__ Tables T;
  load_huff(T, tab);
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n_sub = st->n_sub;
  if (s >= n_sub) return;
  const Sub sub = subs[s];
  const unsigned long long entry = ecur[s];
  unsigned long long x;
  if (entry == used[s]) {                                  // decoded from this entry in an earlier pass
    x = exits[s];
  } else {
    S4 acc = {};
    x = run_sub<false>(T, g, U, sub.z, entry, acc, S4{}, 0, 0, 0, nullptr, st);
    agg[s] = acc;
    exits[s] = x;
    used[s] = entry;
  }
  if (sub.head) enext[s] = entry;
  // a predecessor that hit an invalid code leaves its successor's entry as it is: at the fixpoint that is either
  // data past an interval's last block or a corrupt stream, which the writing pass reports
  if (s + 1 < n_sub && !subs[s + 1].head) {
    const unsigned long long e = x == kDead ? ecur[s + 1] : x;
    enext[s + 1] = e;
    if (e != ecur[s + 1]) st->changed[pass] = 1;
  }
}

__global__ void __launch_bounds__(128) write_pass(const Tables* tab, Geo g, const uint8_t* U, const Sub* subs,
                                                  const uint2* iv_se, State* st, const unsigned long long* entry,
                                                  const S4* agg, int16_t* coef, int last_pass) {
  if (st->changed[last_pass] != 0) {
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicOr(&st->status, ST_CONVERGE);
    return;
  }
  if (st->status) return;
  __shared__ Tables T;
  load_huff(T, tab);
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= st->n_sub) return;
  const Sub sub = subs[s];
  const S4 carry = sub.head ? S4{} : agg[s - 1];            // agg: inclusive per-interval sums
  const long long total_mcus = (long long)g.mcus_x * g.mcus_y;
  const long long mcu0 = (long long)sub.iv * g.ri;
  const long long expected = min((long long)g.ri, total_mcus - mcu0) * g.bpm;
  S4 acc = {};
  run_sub<true>(T, g, U, sub.z, entry[s], acc, carry, expected, mcu0, iv_se[sub.iv].y, coef, st);
}

// ------------------------------------------------------------------------------------------------ device: IDCT
// jpeg_idct_islow: 8 threads per block (one column in pass 1, one row in pass 2), 32 blocks per CTA.
// Pillow's libjpeg-turbo runs either the C version (64-bit products, masked range-limit table) or a SIMD one (16-bit
// dequantisation, saturating packs after each pass).  The two give the same bytes while every dequantised coefficient
// and every pass-1 value fits in int16 and every output before the level shift lies in [-512, 511], where the C table
// clamps like the SIMD saturation.  Real encoders stay far inside that window; a block that leaves it sets ST_RANGE,
// so the caller takes Pillow's own decode.  The arithmetic is 64-bit, as the C version's, so the checks see true values.
constexpr int kIdctBlocks = 32;

__device__ __forceinline__ void idct_1d(long long s0, long long s1, long long s2, long long s3, long long s4,
                                        long long s5, long long s6, long long s7, long long* o) {
  long long z1 = (s2 + s6) * 4433;                   // FIX_0_541196100
  const long long tmp2 = z1 + s6 * -15137, tmp3 = z1 + s2 * 6270;
  const long long tmp0 = (s0 + s4) * 8192, tmp1 = (s0 - s4) * 8192;
  const long long t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  long long t0 = s7, t1 = s5, t2 = s3, t3 = s1;
  z1 = t0 + t3;
  long long z2 = t1 + t2, z3 = t0 + t2, z4 = t1 + t3;
  const long long z5 = (z3 + z4) * 9633;
  t0 *= 2446; t1 *= 16819; t2 *= 25172; t3 *= 12299;
  z1 *= -7373; z2 *= -20995; z3 = z3 * -16069 + z5; z4 = z4 * -3196 + z5;
  t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
  o[0] = t10 + t3; o[7] = t10 - t3; o[1] = t11 + t2; o[6] = t11 - t2;
  o[2] = t12 + t1; o[5] = t12 - t1; o[3] = t13 + t0; o[4] = t13 - t0;
}

__global__ void __launch_bounds__(256) idct_islow(const Tables* tab, Geo g, const int16_t* coef, uint8_t* pix,
                                                  long long n_blocks, State* st) {
  if (st->status) return;
  __shared__ int ws[kIdctBlocks][64];
  __shared__ uint16_t q[3][64];
  for (int i = threadIdx.x; i < 3 * 64; i += blockDim.x) q[i / 64][i % 64] = tab->qt[g.tq[i / 64]][i % 64];
  __syncthreads();
  const int lb = threadIdx.x >> 3, j = threadIdx.x & 7;
  const long long blk = (long long)blockIdx.x * kIdctBlocks + lb;
  const bool live = blk < n_blocks;
  int c = 0;
  long long local = blk;
  if (live) {
    while (c < 2 && local >= (long long)g.bw[c] * g.bh[c]) local -= (long long)g.bw[c] * g.bh[c], ++c;
    const int16_t* x = coef + g.coef_off[c] + local * 64;
    long long in[8], o[8];
    bool out_of_range = false;
    for (int r = 0; r < 8; ++r) {
      in[r] = (long long)x[r * 8 + j] * q[c][r * 8 + j];
      out_of_range |= in[r] < -32768 || in[r] > 32767;
    }
    idct_1d(in[0], in[1], in[2], in[3], in[4], in[5], in[6], in[7], o);
    for (int r = 0; r < 8; ++r) {
      const long long v = (o[r] + (1 << 10)) >> 11;
      out_of_range |= v < -32768 || v > 32767;
      ws[lb][r * 8 + j] = (int)v;
    }
    if (out_of_range) atomicOr(&st->status, ST_RANGE);
  }
  __syncthreads();
  if (!live) return;
  const int* w = ws[lb] + j * 8;
  long long o[8];
  idct_1d(w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7], o);
  uint32_t lo = 0, hi = 0;
  bool out_of_range = false;
  for (int i = 0; i < 8; ++i) {
    const long long y = (o[i] + (1 << 17)) >> 18;
    out_of_range |= y < -512 || y > 511;
    const int idx = (int)(y & 1023);                      // libjpeg's post-IDCT range-limit table
    const uint32_t v = idx < 128 ? idx + 128 : (idx < 512 ? 255 : (idx < 896 ? 0 : idx - 896));
    if (i < 4) lo |= v << (8 * i); else hi |= v << (8 * (i - 4));
  }
  if (out_of_range) atomicOr(&st->status, ST_RANGE);
  const long long by = local / g.bw[c], bx = local % g.bw[c];
  uint8_t* dst = pix + g.pix_off[c] + (by * 8 + j) * (long long)g.bw[c] * 8 + bx * 8;
  *reinterpret_cast<uint2*>(dst) = make_uint2(lo, hi);
}

// ------------------------------------------------------------------------------------------------ device: colour
// jdsample.c's fancy upsampling (h2v1, h2v2) over the true downsampled extents, replication when that width is 2 or
// less (jinit_upsampler), then jdcolor.c's ycc_rgb_convert.
__device__ __forceinline__ int chroma(const uint8_t* P, int pitch, int y, int x, const Geo& g) {
  if (g.hY == 1) return P[(long long)y * pitch + x];
  const int dw = (g.W + 1) >> 1, c = x >> 1;
  const int r = g.vY == 2 ? y >> 1 : y;
  const uint8_t* row = P + (long long)r * pitch;
  if (dw <= 2) return row[c];
  if (g.vY == 1) {
    const int v = row[c];
    if (!(x & 1)) return c == 0 ? v : (3 * v + row[c - 1] + 1) >> 2;
    return c == dw - 1 ? v : (3 * v + row[c + 1] + 2) >> 2;
  }
  const int dh = (g.H + 1) >> 1;
  const int nr = (y & 1) ? min(r + 1, dh - 1) : max(r - 1, 0);
  const uint8_t* nb = P + (long long)nr * pitch;
  const int cs = 3 * row[c] + nb[c];
  if (!(x & 1)) return c == 0 ? (4 * cs + 8) >> 4 : (3 * cs + 3 * row[c - 1] + nb[c - 1] + 8) >> 4;
  return c == dw - 1 ? (4 * cs + 7) >> 4 : (3 * cs + 3 * row[c + 1] + nb[c + 1] + 7) >> 4;
}

__global__ void __launch_bounds__(256) ycc_to_rgb(Geo g, const uint8_t* pix, uint8_t* dst, long long rs, long long ps,
                                                  long long cs, const State* st) {
  if (st->status) return;
  const long long n = (long long)g.W * g.H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(i / g.W), x = (int)(i % g.W);
    const int Y = pix[g.pix_off[0] + (long long)y * g.bw[0] * 8 + x];
    const int cb = chroma(pix + g.pix_off[1], g.bw[1] * 8, y, x, g) - 128;
    const int cr = chroma(pix + g.pix_off[2], g.bw[2] * 8, y, x, g) - 128;
    const int r = Y + ((91881 * cr + 32768) >> 16);
    const int gg = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
    const int b = Y + ((116130 * cb + 32768) >> 16);
    uint8_t* o = dst + y * rs + x * ps;
    o[0] = (uint8_t)min(max(r, 0), 255);
    o[cs] = (uint8_t)min(max(gg, 0), 255);
    o[2 * cs] = (uint8_t)min(max(b, 0), 255);
  }
}

unsigned grid(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

}  // namespace

extern "C" {

gp_status gp_jpeg_probe(const uint8_t* data, size_t nbytes, int* H, int* W, int64_t* workspace_bytes) {
  return gp::guarded_call([&]() {
    const Header hd = parse(data, nbytes);
    const Layout y = plan(hd, nbytes);
    if (H) *H = hd.H;
    if (W) *W = hd.W;
    if (workspace_bytes) *workspace_bytes = (int64_t)y.total;
  });
}

gp_status gp_jpeg_decode(const uint8_t* data_host, size_t nbytes, void* workspace_dev, int64_t workspace_bytes,
                         uint8_t* dst_dev, int64_t row_stride, int64_t pixel_stride, int64_t channel_stride,
                         void* stream) {
  return gp::guarded_call([&]() {
    const Header hd = parse(data_host, nbytes);
    const Layout y = plan(hd, nbytes);
    GP_REQUIRE(workspace_dev && workspace_bytes >= (int64_t)y.total, "workspace too small");
    GP_REQUIRE(dst_dev, "no output buffer");
    const Geo& g = y.g;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    uint8_t* ws = static_cast<uint8_t*>(workspace_dev);
    auto at = [&](size_t o) { return ws + o; };
    const uint8_t* E = at(y.o_file) + hd.start;
    const Tables* tab = reinterpret_cast<const Tables*>(at(y.o_tab));
    State* st = reinterpret_cast<State*>(at(y.o_state));
    S4* chunks = reinterpret_cast<S4*>(at(y.o_chunk));
    uint8_t* U = at(y.o_u);
    uint32_t* rst = reinterpret_cast<uint32_t*>(at(y.o_rst));
    S4* iv = reinterpret_cast<S4*>(at(y.o_iv));
    uint2* iv_se = reinterpret_cast<uint2*>(at(y.o_iv_se));
    Sub* subs = reinterpret_cast<Sub*>(at(y.o_sub));
    unsigned long long* e[2] = {reinterpret_cast<unsigned long long*>(at(y.o_e0)),
                                reinterpret_cast<unsigned long long*>(at(y.o_e1))};
    S4* agg = reinterpret_cast<S4*>(at(y.o_agg));
    int16_t* coef = reinterpret_cast<int16_t*>(at(y.o_coef));
    uint8_t* pix = at(y.o_pix);

    State init;
    memset(&init, 0, sizeof init);
    init.end = (int)y.L;
    GP_CUDA(cudaMemcpyAsync(at(y.o_file), data_host, nbytes, cudaMemcpyHostToDevice, s));
    GP_CUDA(cudaMemcpyAsync(at(y.o_tab), &hd.t, sizeof(Tables), cudaMemcpyHostToDevice, s));
    GP_CUDA(cudaMemcpyAsync(st, &init, sizeof init, cudaMemcpyHostToDevice, s));
    GP_CUDA(cudaMemsetAsync(U, 0, y.o_rst - y.o_u, s));
    GP_CUDA(cudaMemsetAsync(rst, 0, (size_t)g.n_int * 4, s));
    GP_CUDA(cudaMemsetAsync(coef, 0, (size_t)y.coef_elems * 2, s));

    find_end<<<grid(y.L, 256 * 16), 256, 0, s>>>(E, y.L, st);
    unstuff_count<<<(unsigned)y.n_chunks, 256, 0, s>>>(E, y.L, st, chunks, at(y.o_chunk_f));
    scan(chunks, at(y.o_chunk_f), y.n_chunks, reinterpret_cast<S4*>(at(y.o_chunk_b)), at(y.o_chunk_bf), s);
    unstuff_write<<<(unsigned)y.n_chunks, 256, 0, s>>>(E, st, chunks, U, rst, g.n_int - 1);
    intervals<<<grid(g.n_int, 256), 256, 0, s>>>(st, chunks, y.n_chunks, rst, g.n_int, iv, at(y.o_iv_f), iv_se);
    scan(iv, at(y.o_iv_f), g.n_int, reinterpret_cast<S4*>(at(y.o_iv_b)), at(y.o_iv_bf), s);
    unsigned long long* used = reinterpret_cast<unsigned long long*>(at(y.o_used));
    unsigned long long* exits = reinterpret_cast<unsigned long long*>(at(y.o_exit));
    subsequences<<<grid(y.n_sub_max, 256), 256, 0, s>>>(st, iv, iv_se, g.n_int, y.n_sub_max, subs, e[0], e[1], used,
                                                          at(y.o_agg_f));
    // passes in batches; a pass after convergence returns at once, and the host stops at the first converged batch
    int last = 0;
    for (int pass = 0; pass < kMaxPasses; pass += kPassBatch) {
      for (int j = pass; j < pass + kPassBatch; ++j)
        sync_pass<<<grid(y.n_sub_max, 128), 128, 0, s>>>(tab, g, U, subs, st, j, e[j & 1], e[(j + 1) & 1], used,
                                                         exits, agg);
      last = pass + kPassBatch - 1;
      int changed = 1;
      GP_CUDA(cudaMemcpyAsync(&changed, &st->changed[last], sizeof changed, cudaMemcpyDeviceToHost, s));
      GP_CUDA(cudaStreamSynchronize(s));
      if (!changed) break;
    }
    scan(agg, at(y.o_agg_f), y.n_sub_max, reinterpret_cast<S4*>(at(y.o_agg_b)), at(y.o_agg_bf), s);
    write_pass<<<grid(y.n_sub_max, 128), 128, 0, s>>>(tab, g, U, subs, iv_se, st, e[0], agg, coef, last);
    idct_islow<<<grid(y.n_blocks, kIdctBlocks), 256, 0, s>>>(tab, g, coef, pix, y.n_blocks, st);
    ycc_to_rgb<<<grid((long long)g.W * g.H, 256), 256, 0, s>>>(g, pix, dst_dev, row_stride, pixel_stride,
                                                              channel_stride, st);
    GP_CUDA(cudaGetLastError());
    State out;
    GP_CUDA(cudaMemcpyAsync(&out, st, sizeof out, cudaMemcpyDeviceToHost, s));
    GP_CUDA(cudaStreamSynchronize(s));
    if (out.status == 0 && out.blocks_done != (unsigned long long)y.n_blocks) out.status = ST_COUNT;
    if (out.status) {
      static const char* why[] = {"unexpected marker or no EOI in the scan", "restart markers out of sequence",
                                  "invalid Huffman code or coefficient run", "entropy-coded data exhausted",
                                  "decode did not converge", "block count differs from the frame's",
                                  "DC coefficient out of range", "subsequence layout overflow",
                                  "IDCT value outside the range libjpeg-turbo's C and SIMD IDCTs agree on"};
      int bit = 0;
      while (!(out.status >> bit & 1)) ++bit;
      throw gp::GpError(GP_ERR_INVALID, std::string("corrupt or undecodable JPEG stream: ") + why[bit]);
    }
  });
}

}  // extern "C"
