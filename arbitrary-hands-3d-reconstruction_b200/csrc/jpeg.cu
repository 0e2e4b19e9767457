// Baseline JPEG decoding on the device (include/acr_b200.h, acr_b200_jpeg_decode): Huffman decoding, islow IDCT,
// fancy upsampling and YCbCr->BGR, bit for bit libjpeg-turbo's defaults (what cv2.imdecode does).
//
// Work split.  A frame's entropy-coded segment is cut into chunks of ACR_B200_JPEG_CHUNK raw bytes, one thread
// each.  A decoder state is (position, z, c): the raw byte and bit of the next code, the coefficient index of the
// block being decoded (0 = its DC is next) and the block's slot in the MCU.  Positions are raw offsets in the
// segment: byte stuffing (FF 00) is skipped when bits are read, and a restart marker, with any FF fill bytes before
// it, is crossed when a decoder at a code boundary finds nothing but padding ones before it.  A chunk's work is
// every code that starts at a position before the chunk's end; its end state is the first code boundary at or past
// that end.
//
//   jpeg_spec_kernel   self-synchronising speculative decoding (Weissenberger & Schmidt, ICPP 2018): the thread of
//                      chunk j guesses a code boundary at the start of chunk j-1 (z = c = 0), decodes through it
//                      to reach the start of chunk j ("from"), then decodes chunk j: its end state and summary
//                      (blocks started, DC sums since the last restart, restarts, errors).  Huffman codes resync
//                      within a few codes, so "from" is almost always the true start.
//   jpeg_sync_kernel   one CTA per frame: chunk j's guess is right when from[j] == end[j-1].  Chunks where it is
//                      not are decoded again from end[j-1] until every start agrees (chunk 0 starts at the true
//                      start, so this ends).  Then a segmented prefix over the chunks gives each chunk its first
//                      block and its DC predictions, and the frame its status.
//   jpeg_write_kernel  every chunk decodes again from its true start and stores its coefficients (int16,
//                      quantised, natural order) into the component planes of blocks.
//   jpeg_idct_kernel   one thread per block: dequantise, islow IDCT, range limit -> component sample planes.
//   jpeg_color_kernel  one thread per pixel: libjpeg-turbo's triangle upsampling of the chroma (h2v1, h2v2, h1v2;
//                      replication for planes at most 2 wide) and the fixed-point YCbCr->BGR tables.
// Multi-scan files (acr_b200_jpeg_decode_scans): jpeg_scan_spec / _sync / _write_kernel run the same scheme over the
// first scans of every file (DC first, AC first, sequential), one sync CTA per scan; jpeg_refine_kernel then applies
// each frame's refinement scans in file order, one CTA per frame: a serial walk finds every block's start from
// nonzero masks, then the CTA decodes the blocks in parallel.
// No kernel uses shared-memory atomics' order in a result, and none uses local memory.
#include "common.cuh"

namespace acr {
namespace {

constexpr int CHUNK = ACR_B200_JPEG_CHUNK;
constexpr int ST_DONE = 1 << 16;   // state flag: the segment's end was reached
constexpr int PENDING = 1 << 30;   // Chunk::err: decode again from `from` (sync kernel)
constexpr int BAD_DESC = 1 << 8;   // status: the descriptor does not fit the buffers

static_assert(sizeof(acr_b200_jpeg_huff) == 1424, "acr_b200_jpeg_huff layout");
static_assert(sizeof(acr_b200_jpeg_frame) == 9112, "acr_b200_jpeg_frame layout");

struct Chunk {
  int2 from;            // x: raw bit position (byte * 8 + bit), y: z | c << 8 | ST_* flags
  int2 end;
  int nblk, dc[3], nres, err;   // summary of the decode from `from`
  int blk0, pred[3];            // blocks started before the chunk, DC predictions at its start
};

__constant__ uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct Args {
  const uint8_t* coded;
  long long coded_bytes;
  const acr_b200_jpeg_frame* frames;
  int n;
  long long max_chunks, max_blocks;
  Chunk* chunks;
  int16_t* coef;
  uint8_t* planes;
  uint8_t* out;
  long long out_bytes;
  int32_t* status;
  // acr_b200_jpeg_decode_scans only (null / 0 in acr_b200_jpeg_decode)
  const acr_b200_jpeg_scan* scans;
  long long max_scans;
  int32_t* scan_status;   // per scan: its descriptor check and the first-scan decode's bits
  unsigned long long* refine_masks;   // per block: nonzero coefficients of a refinement scan's band
  int4* refine_starts;                // per block: the bit reader where its refinement codes start, and the EOB
                                      // run left
};

// The frame's block geometry and output range fit the buffers.
__device__ bool frame_geometry_ok(const Args& a, const acr_b200_jpeg_frame& f) {
  if (f.ncomp != 1 && f.ncomp != 3) return false;
  if (f.H < 1 || f.W < 1 || f.out_offset < 0 || f.out_offset + 3LL * f.H * f.W > a.out_bytes) return false;
  if (f.bpm < 1 || f.bpm > 6 || f.mcus_x < 1 || f.mcus_y < 1 || f.block_begin < 0 || f.coef_offset != f.block_begin ||
      (long long)f.mcus_x * f.mcus_y * f.bpm != f.n_blocks || (long long)f.block_begin + f.n_blocks > a.max_blocks)
    return false;
  long long planes = 0;
  for (int c = 0; c < f.ncomp; ++c) {
    if (f.comp_h[c] < 1 || f.comp_h[c] > 2 || f.comp_v[c] < 1 || f.comp_v[c] > 2 || f.comp_block0[c] != planes ||
        f.comp_bw[c] != f.mcus_x * f.comp_h[c] || f.comp_bh[c] != f.mcus_y * f.comp_v[c] || f.comp_w[c] < 1 ||
        f.comp_hgt[c] < 1 || f.comp_w[c] > 8 * f.comp_bw[c] || f.comp_hgt[c] > 8 * f.comp_bh[c])
      return false;
    planes += (long long)f.comp_bw[c] * f.comp_bh[c];
  }
  if (planes != f.n_blocks) return false;
  for (int k = 0; k < f.bpm; ++k) {
    const int c = f.slot_comp[k];
    if (c < 0 || c >= f.ncomp || f.slot_dy[k] < 0 || f.slot_dy[k] >= f.comp_v[c] || f.slot_dx[k] < 0 ||
        f.slot_dx[k] >= f.comp_h[c])
      return false;
  }
  return true;
}

// A single-scan descriptor whose ranges do not fit the buffers is not decoded (status BAD_DESC, set by the sync
// kernel).
__device__ bool frame_ok(const Args& a, const acr_b200_jpeg_frame& f) {
  if (f.n_scans != 0 || f.coded_len < 0 || f.coded_len >= ACR_B200_JPEG_MAX_SCAN_BYTES || f.coded_offset < 0 ||
      f.coded_offset + f.coded_len > a.coded_bytes)
    return false;
  if (f.chunk_begin < 0 || f.n_chunks != (f.coded_len + CHUNK - 1) / CHUNK + (f.coded_len == 0) ||
      (long long)f.chunk_begin + f.n_chunks > a.max_chunks)
    return false;
  return frame_geometry_ok(a, f);
}

// Last frame whose first index (chunk_begin, block_begin or out_offset / 3) is <= g.
template <typename Key>
__device__ int find_frame(const acr_b200_jpeg_frame* fr, int n, long long g, Key key) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (key(fr[mid]) <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}

struct Summary {
  int nblk, dc[3], nres, err;
};

// Where the write pass stores: the frame's coefficient blocks, the block being decoded and the DC predictions.
struct Store {
  int16_t* coef;
  int cur;        // frame-relative index of the block being decoded (-1 before the first DC of the chunk)
  int pred[3];
  int16_t* blk;   // its coefficients, or nullptr when it is out of range
};

struct Decoder {
  const uint8_t* seg;
  int len;
  int b, o;   // next unread bit: raw byte b (a data byte), bit o (0 = MSB)
  int z, c, flags;

  __device__ int2 state() const { return make_int2(b * 8 + o, z | (c << 8) | flags); }
  __device__ void set(int2 s) {
    b = s.x >> 3;
    o = s.x & 7;
    z = s.y & 0xFF;
    c = (s.y >> 8) & 0xFF;
    flags = s.y & ST_DONE;
  }
  // A guessed code boundary at raw byte s: step off the second byte of a stuffed FF 00 or of a marker.
  __device__ __forceinline__ void guess(int s) {
    if (s > 0 && s < len && seg[s - 1] == 0xFF) ++s;
    b = s;
    o = 0;
    z = c = flags = 0;
  }
  // 32 bits from the current position, MSB first, zero past the data; avail = valid bits (<= 32); stop = raw
  // offset of the marker or segment end that cut the window (-1 if none did).
  __device__ __forceinline__ uint32_t peek(int& avail, int& stop) const {
    unsigned long long acc = 0;
    int n = 0, q = b;
    stop = -1;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      if (stop < 0) {
        if (q >= len) {
          stop = q;
        } else {
          const uint32_t x = seg[q];
          if (x == 0xFF && !(q + 1 < len && seg[q + 1] == 0)) {
            stop = q;
          } else {
            q += x == 0xFF ? 2 : 1;
            acc |= (unsigned long long)x << (56 - n);
            n += 8;
          }
        }
      }
    }
    avail = min(max(n - o, 0), 32);
    return (uint32_t)((acc << o) >> 32);
  }
  __device__ __forceinline__ void advance(int bits) {
    o += bits;
    while (o >= 8) {
      b += seg[b] == 0xFF ? 2 : 1;
      o -= 8;
    }
  }
  // An error is recorded, and decoding goes on from a guess one byte on: a decoder that started at a wrong guess
  // must be able to resynchronise (a stop would hand its successors a wrong start, chunk after chunk).  From the
  // true start of valid data no error happens, so the bits only ever reach the status of a corrupt frame.
  __device__ __forceinline__ void fail(Summary& s, int why) {
    s.err |= why;
    guess(b + 1);
  }
};

// One Huffman code from the 32-bit window w -> length (0 if no code matches), symbol.
__device__ __forceinline__ int huff(const acr_b200_jpeg_huff& t, uint32_t w, int& sym) {
  const int e = t.lut[w >> 23];
  if (e) {
    sym = e & 0xFF;
    return e >> 8;
  }
  int l = 10;
  while (l <= 16 && (int)(w >> (32 - l)) > t.maxcode[l]) ++l;
  if (l > 16) return 0;
  sym = t.huffval[((int)(w >> (32 - l)) + t.valoff[l]) & 0xFF];
  return l;
}

// a[k] += v with a constant-index select, so that small arrays stay in registers
__device__ __forceinline__ void add_at(int* a, int k, int v) {
  if (k == 0) a[0] += v; else if (k == 1) a[1] += v; else a[2] += v;
}
__device__ __forceinline__ int get_at(const int* a, int k) { return k == 0 ? a[0] : k == 1 ? a[1] : a[2]; }

__device__ __forceinline__ int extend(uint32_t v, int s) { return v < (1u << (s - 1)) ? (int)v - (1 << s) + 1 : (int)v; }

// Decode codes that start before raw byte `end_b` (the whole rest of the segment if end_b >= len).  WRITE: also
// store coefficients (st) and check restart placement against the frame's block numbering.
template <bool WRITE>
__device__ __forceinline__ void run(Decoder& d, const acr_b200_jpeg_frame& f, int end_b, Summary& s, Store* st) {
  while (!d.flags && d.b < end_b) {
    int avail, stop;
    const uint32_t w = d.peek(avail, stop);
    if (avail < 8 && (avail == 0 || (w >> (32 - avail)) == (1u << avail) - 1)) {   // only padding before a marker
      if (d.z != 0 || d.c != 0) { d.fail(s, ACR_B200_JPEG_TRUNCATED); continue; }
      // a marker may follow any number of FF fill bytes (T.81 B.1.1.2); fill bytes up to the segment's end
      // precede its EOI
      int q = stop;
      while (q + 1 < d.len && d.seg[q + 1] == 0xFF) ++q;
      if (q + 1 >= d.len) { d.flags |= ST_DONE; break; }
      const int m = d.seg[q + 1];
      if (m < 0xD0 || m > 0xD7) {   // resume past the fill run: a decoder crosses it once
        d.b = q;
        d.fail(s, ACR_B200_JPEG_BAD_MARKER);
        continue;
      }
      if (WRITE) {   // the interval before must be `restart` whole MCUs, and the marker the next in sequence
        const int next = st->cur + 1, per = f.restart * f.bpm;
        if (per == 0 || next == 0 || next % per != 0 || ((next / per - 1) & 7) != m - 0xD0)
          s.err |= ACR_B200_JPEG_BAD_RESTART;
        st->pred[0] = st->pred[1] = st->pred[2] = 0;
      }
      d.b = q + 2;
      d.o = 0;
      s.nres += 1;
      s.dc[0] = s.dc[1] = s.dc[2] = 0;
      continue;
    }
    const int comp = f.slot_comp[d.c];
    int sym, l;
    if (d.z == 0) {
      l = huff(f.dc[comp], w, sym);
      if (l == 0 || sym > 15) { d.fail(s, ACR_B200_JPEG_BAD_CODE); continue; }
      if (l + sym > avail) { d.fail(s, ACR_B200_JPEG_TRUNCATED); continue; }
      const int diff = sym ? extend((w << l) >> (32 - sym), sym) : 0;
      d.advance(l + sym);
      s.nblk += 1;
      add_at(s.dc, comp, diff);
      d.z = 1;
      if (WRITE) {
        st->cur += 1;
        add_at(st->pred, comp, diff);
        st->blk = nullptr;
        if (st->cur < f.n_blocks) {
          const int mcu = st->cur / f.bpm, k = st->cur - mcu * f.bpm, my = mcu / f.mcus_x, mx = mcu - my * f.mcus_x;
          const int by = my * f.comp_v[comp] + f.slot_dy[k], bx = mx * f.comp_h[comp] + f.slot_dx[k];
          st->blk = st->coef + 64LL * (f.coef_offset + f.comp_block0[comp] + (long long)by * f.comp_bw[comp] + bx);
          st->blk[0] = (int16_t)get_at(st->pred, comp);
        }
      }
    } else {
      l = huff(f.ac[comp], w, sym);
      if (l == 0) { d.fail(s, ACR_B200_JPEG_BAD_CODE); continue; }
      const int r = sym >> 4, sz = sym & 15;
      if (l + sz > avail) { d.fail(s, ACR_B200_JPEG_TRUNCATED); continue; }
      if (sz) {
        d.z += r;
        if (d.z > 63) { d.fail(s, ACR_B200_JPEG_BAD_CODE); continue; }
        if (WRITE && st->blk) st->blk[kZigzag[d.z]] = (int16_t)extend((w << l) >> (32 - sz), sz);
        d.z += 1;
      } else {
        d.z = r == 15 ? d.z + 16 : 64;
      }
      d.advance(l + sz);
    }
    if (d.z >= 64) {
      d.z = 0;
      d.c = d.c + 1 == f.bpm ? 0 : d.c + 1;
    }
  }
}

// f: a frame or a scan descriptor
template <typename Desc>
__device__ int chunk_end(const Desc& f, int j) {
  return j + 1 == f.n_chunks ? 0x7fffffff : (j + 1) * CHUNK;
}

// 64 registers: left to itself ptxas picks 40 for occupancy and spills the decoder state to local memory
__global__ void __maxnreg__(64) jpeg_spec_kernel(Args a) {
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (g >= a.max_chunks) return;
  const int fi = find_frame(a.frames, a.n, g, [](const acr_b200_jpeg_frame& f) { return (long long)f.chunk_begin; });
  const acr_b200_jpeg_frame& f = a.frames[fi];
  const int j = (int)(g - f.chunk_begin);
  if (j < 0 || j >= f.n_chunks || !frame_ok(a, f)) return;
  Decoder d{a.coded + f.coded_offset, f.coded_len, 0, 0, 0, 0, 0};
  Summary s{};
  Chunk& ch = a.chunks[g];
  if (j > 0) {   // warm up from a guess one chunk back to reach the start of chunk j
    d.guess((j - 1) * CHUNK);
    run<false>(d, f, j * CHUNK, s, nullptr);
    s = Summary{};
  }
  ch.from = d.state();
  run<false>(d, f, chunk_end(f, j), s, nullptr);
  ch.end = d.state();
  ch.nblk = s.nblk;
  ch.dc[0] = s.dc[0], ch.dc[1] = s.dc[1], ch.dc[2] = s.dc[2];
  ch.nres = s.nres;
  ch.err = s.err;
}

constexpr int SYNC_THREADS = 512;

__device__ __forceinline__ bool same(int2 p, int2 q) { return p.x == q.x && p.y == q.y; }

// Synchronise the n chunks of one frame or scan (one CTA): Jacobi rounds until every chunk starts where its
// predecessor ends, then a segmented prefix of the block counts and DC sums.  u.run(d, j, s) decodes chunk j from the
// state d was set to; the status bits go to *status.
template <typename Unit>
__device__ __forceinline__ void sync_chunks(const Unit& u, Chunk* ch, int n, int n_blocks, int32_t* status) {
  const int tid = threadIdx.x;
  while (true) {   // Jacobi rounds: after round k, chunks 0..k have their true start
    int any = 0;
    for (int j = 1 + tid; j < n; j += SYNC_THREADS) {
      if (!same(ch[j].from, ch[j - 1].end)) {
        ch[j].from = ch[j - 1].end;
        ch[j].err |= PENDING;
        any = 1;
      }
    }
    if (!__syncthreads_or(any)) break;
    for (int j = 1 + tid; j < n; j += SYNC_THREADS) {
      if (ch[j].err & PENDING) {
        Decoder d = u.decoder();
        d.set(ch[j].from);
        Summary s{};
        u.run(d, j, s);
        ch[j].end = d.state();
        ch[j].nblk = s.nblk;
        ch[j].dc[0] = s.dc[0], ch[j].dc[1] = s.dc[1], ch[j].dc[2] = s.dc[2];
        ch[j].nres = s.nres;
        ch[j].err = s.err;
      }
    }
    __syncthreads();
  }
  // exclusive segmented prefix of (blocks started, DC sums; a restart clears the sums) over the chunks
  __shared__ int sn[SYNC_THREADS], sd[3][SYNC_THREADS], sr[SYNC_THREADS];
  __shared__ int err_all;
  if (tid == 0) err_all = 0;
  const int per = (n + SYNC_THREADS - 1) / SYNC_THREADS, j0 = min(n, tid * per), j1 = min(n, j0 + per);
  int nb = 0, d0 = 0, d1 = 0, d2 = 0, rs = 0, err = 0;
  for (int j = j0; j < j1; ++j) {
    const Chunk& c = ch[j];
    nb += c.nblk;
    if (c.nres) d0 = d1 = d2 = 0, rs = 1;
    d0 += c.dc[0], d1 += c.dc[1], d2 += c.dc[2];
    err |= c.err;
  }
  sn[tid] = nb, sd[0][tid] = d0, sd[1][tid] = d1, sd[2][tid] = d2, sr[tid] = rs;
  __syncthreads();
  atomicOr(&err_all, err);
  for (int off = 1; off < SYNC_THREADS; off <<= 1) {   // inclusive Hillis-Steele scan
    int pn = 0, p0 = 0, p1 = 0, p2 = 0, pr = 0;
    if (tid >= off) pn = sn[tid - off], p0 = sd[0][tid - off], p1 = sd[1][tid - off], p2 = sd[2][tid - off], pr = sr[tid - off];
    __syncthreads();
    if (tid >= off) {
      sn[tid] += pn;
      if (!sr[tid]) sd[0][tid] += p0, sd[1][tid] += p1, sd[2][tid] += p2;
      sr[tid] |= pr;
    }
    __syncthreads();
  }
  nb = tid ? sn[tid - 1] : 0;
  d0 = tid ? sd[0][tid - 1] : 0, d1 = tid ? sd[1][tid - 1] : 0, d2 = tid ? sd[2][tid - 1] : 0;
  for (int j = j0; j < j1; ++j) {
    Chunk& c = ch[j];
    c.blk0 = nb;
    c.pred[0] = d0, c.pred[1] = d1, c.pred[2] = d2;
    nb += c.nblk;
    if (c.nres) d0 = d1 = d2 = 0;
    d0 += c.dc[0], d1 += c.dc[1], d2 += c.dc[2];
  }
  if (tid == SYNC_THREADS - 1) {
    const int total = sn[SYNC_THREADS - 1];
    int st = err_all & ~PENDING;
    if (!(ch[n - 1].end.y & ST_DONE)) st |= ACR_B200_JPEG_TRUNCATED;
    if (total < n_blocks) st |= ACR_B200_JPEG_TRUNCATED;
    if (total > n_blocks) st |= ACR_B200_JPEG_BAD_LENGTH;
    *status = st;
  }
}

struct FrameUnit {
  const Args& a;
  const acr_b200_jpeg_frame& f;
  __device__ Decoder decoder() const { return Decoder{a.coded + f.coded_offset, f.coded_len, 0, 0, 0, 0, 0}; }
  __device__ void run(Decoder& d, int j, Summary& s) const { acr::run<false>(d, f, chunk_end(f, j), s, nullptr); }
};

// one CTA per frame, so occupancy does not matter: min blocks 1 keeps ptxas from capping the registers at 32 and
// spilling the decoder state to local memory
__global__ void __launch_bounds__(SYNC_THREADS, 1) jpeg_sync_kernel(Args a) {
  const acr_b200_jpeg_frame& f = a.frames[blockIdx.x];
  const int tid = threadIdx.x;
  if (f.ncomp == 0) {   // decoded elsewhere (host fallback)
    if (tid == 0) a.status[blockIdx.x] = 0;
    return;
  }
  if (f.n_scans != 0 && a.scans) return;   // a multi-scan frame: its status comes from jpeg_refine_kernel
  if (!frame_ok(a, f)) {
    if (tid == 0) a.status[blockIdx.x] = BAD_DESC;
    return;
  }
  sync_chunks(FrameUnit{a, f}, a.chunks + f.chunk_begin, f.n_chunks, f.n_blocks, a.status + blockIdx.x);
}

__global__ void __maxnreg__(64) jpeg_write_kernel(Args a) {
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (g >= a.max_chunks) return;
  const int fi = find_frame(a.frames, a.n, g, [](const acr_b200_jpeg_frame& f) { return (long long)f.chunk_begin; });
  const acr_b200_jpeg_frame& f = a.frames[fi];
  const int j = (int)(g - f.chunk_begin);
  if (f.ncomp == 0 || f.n_scans != 0 || j < 0 || j >= f.n_chunks || a.status[fi] != 0) return;   // status 0
                                                                                                    // implies frame_ok
  const Chunk& ch = a.chunks[g];
  Decoder d{a.coded + f.coded_offset, f.coded_len, 0, 0, 0, 0, 0};
  d.set(ch.from);
  Store st{a.coef, ch.blk0 - 1, {ch.pred[0], ch.pred[1], ch.pred[2]}, nullptr};
  if (d.z > 0 && st.cur >= 0 && st.cur < f.n_blocks) {   // the chunk starts inside a block begun before it
    const int comp = f.slot_comp[d.c];
    const int mcu = st.cur / f.bpm, k = st.cur - mcu * f.bpm, my = mcu / f.mcus_x, mx = mcu - my * f.mcus_x;
    const int by = my * f.comp_v[comp] + f.slot_dy[k], bx = mx * f.comp_h[comp] + f.slot_dx[k];
    st.blk = st.coef + 64LL * (f.coef_offset + f.comp_block0[comp] + (long long)by * f.comp_bw[comp] + bx);
  }
  Summary s{};
  run<true>(d, f, chunk_end(f, j), s, &st);
  if (s.err & ACR_B200_JPEG_BAD_RESTART) atomicOr(a.status + fi, ACR_B200_JPEG_BAD_RESTART);
}

// ---- multi-scan files (acr_b200_jpeg_decode_scans) -----------------------------------------------------------------
// A scan descriptor that does not fit its frame or the buffers is not decoded (scan status BAD_DESC).
__device__ bool scan_ok(const Args& a, const acr_b200_jpeg_scan& s) {
  if (s.frame < 0 || s.frame >= a.n || s.ncomp < 1 || s.ncomp > 3) return false;
  const acr_b200_jpeg_frame& f = a.frames[s.frame];
  if (f.n_scans < 1 || s.ncomp > f.ncomp || !frame_geometry_ok(a, f)) return false;
  if (f.coded_offset < 0 || f.coded_len < 0 || f.coded_offset + f.coded_len > a.coded_bytes || s.coded_len < 0 ||
      s.coded_len >= ACR_B200_JPEG_MAX_SCAN_BYTES || s.coded_offset < f.coded_offset ||
      s.coded_offset + s.coded_len > f.coded_offset + f.coded_len)
    return false;
  if (f.chunk_begin < 0 || f.n_chunks < 1 || (long long)f.chunk_begin + f.n_chunks > a.max_chunks ||
      s.n_chunks != (s.coded_len + CHUNK - 1) / CHUNK + (s.coded_len == 0) || s.chunk_begin < f.chunk_begin ||
      (long long)s.chunk_begin + s.n_chunks > (long long)f.chunk_begin + f.n_chunks)
    return false;
  if (s.al < 0 || s.al > 13 || s.ah < 0 || (s.ah != 0 && s.al != s.ah - 1) || s.ss < 0 || s.se < s.ss || s.se > 63)
    return false;
  if (s.ss == 0 && s.se != 0 && !(s.se == 63 && s.ah == 0 && s.al == 0)) return false;   // DC or sequential
  if (s.ss > 0 && s.ncomp != 1) return false;
  if (s.restart < 0 || s.mcus_x < 1 || s.mcus_y < 1 || s.bpm < 1 || s.bpm > 6 ||
      (long long)s.mcus_x * s.mcus_y * s.bpm != s.n_blocks || s.n_blocks > f.n_blocks)
    return false;
  if (s.ncomp > 1) {
    if (s.mcus_x != f.mcus_x || s.mcus_y != f.mcus_y) return false;
    for (int k = 0; k < s.bpm; ++k) {
      const int c = s.slot_comp[k];
      if (c < 0 || c >= f.ncomp || s.slot_dy[k] < 0 || s.slot_dy[k] >= f.comp_v[c] || s.slot_dx[k] < 0 ||
          s.slot_dx[k] >= f.comp_h[c])
        return false;
    }
    return true;
  }
  const int c = s.slot_comp[0];
  return s.bpm == 1 && c >= 0 && c < f.ncomp && s.slot_dy[0] == 0 && s.slot_dx[0] == 0 && s.mcus_x <= f.comp_bw[c] &&
         s.mcus_y <= f.comp_bh[c];
}

// Block k of scan s (nullptr past its blocks).  A one-component scan's blocks are its component's, in raster order.
__device__ __forceinline__ int16_t* scan_block(int16_t* coef, const acr_b200_jpeg_scan& s,
                                               const acr_b200_jpeg_frame& f, int k) {
  if (k >= s.n_blocks) return nullptr;
  const int mcu = k / s.bpm, slot = k - mcu * s.bpm, my = mcu / s.mcus_x, mx = mcu - my * s.mcus_x;
  const int c = s.slot_comp[slot];
  const int by = s.ncomp > 1 ? my * f.comp_v[c] + s.slot_dy[slot] : my;
  const int bx = s.ncomp > 1 ? mx * f.comp_h[c] + s.slot_dx[slot] : mx;
  return coef + 64LL * (f.coef_offset + f.comp_block0[c] + (long long)by * f.comp_bw[c] + bx);
}

struct ScanStore {
  int16_t* coef;
  int cur;        // blocks of the scan finished before the one being decoded
  int pred[3];
  int16_t* blk;   // the block being decoded, or nullptr
};

// run() for a first scan (ah == 0): DC first (ss = se = 0), AC first (ss > 0, one component) or sequential (0..63).
// The state's z is 0 at a block's start and otherwise the next coefficient; an EOBn code ends its whole run of blocks
// at once, so no run is carried from one chunk to the next.  Blocks are counted when they end.
template <bool WRITE>
__device__ __forceinline__ void run_scan(Decoder& d, const acr_b200_jpeg_scan& sc, const acr_b200_jpeg_frame& f,
                                         int end_b, Summary& s, ScanStore* st) {
  while (!d.flags && d.b < end_b) {
    int avail, stop;
    const uint32_t w = d.peek(avail, stop);
    if (avail < 8 && (avail == 0 || (w >> (32 - avail)) == (1u << avail) - 1)) {   // only padding before a marker
      if (d.z != 0 || d.c != 0) { d.fail(s, ACR_B200_JPEG_TRUNCATED); continue; }
      int q = stop;
      while (q + 1 < d.len && d.seg[q + 1] == 0xFF) ++q;
      if (q + 1 >= d.len) { d.flags |= ST_DONE; break; }
      const int m = d.seg[q + 1];
      if (m < 0xD0 || m > 0xD7) {
        d.b = q;
        d.fail(s, ACR_B200_JPEG_BAD_MARKER);
        continue;
      }
      if (WRITE) {   // the interval before must be `restart` whole MCUs, and the marker the next in sequence
        const int next = st->cur, per = sc.restart * sc.bpm;
        if (per == 0 || next == 0 || next % per != 0 || ((next / per - 1) & 7) != m - 0xD0)
          s.err |= ACR_B200_JPEG_BAD_RESTART;
        st->pred[0] = st->pred[1] = st->pred[2] = 0;
      }
      d.b = q + 2;
      d.o = 0;
      s.nres += 1;
      s.dc[0] = s.dc[1] = s.dc[2] = 0;
      continue;
    }
    const int comp = sc.slot_comp[d.c];
    int sym, l, ended = 1;
    if (d.z == 0 && sc.ss == 0) {
      l = huff(sc.dc[comp], w, sym);
      if (l == 0 || sym > 15) { d.fail(s, ACR_B200_JPEG_BAD_CODE); continue; }
      if (l + sym > avail) { d.fail(s, ACR_B200_JPEG_TRUNCATED); continue; }
      const int diff = sym ? extend((w << l) >> (32 - sym), sym) : 0;
      d.advance(l + sym);
      add_at(s.dc, comp, diff);
      if (WRITE) {
        add_at(st->pred, comp, diff);
        st->blk = scan_block(st->coef, sc, f, st->cur);
        if (st->blk) st->blk[0] = (int16_t)(get_at(st->pred, comp) * (1 << sc.al));
      }
      d.z = sc.se == 0 ? 64 : 1;
    } else {
      if (d.z == 0) {
        d.z = sc.ss;
        if (WRITE) st->blk = scan_block(st->coef, sc, f, st->cur);
      }
      l = huff(sc.ac[comp], w, sym);
      if (l == 0) { d.fail(s, ACR_B200_JPEG_BAD_CODE); continue; }
      const int r = sym >> 4, sz = sym & 15;
      if (sz) {
        if (l + sz > avail) { d.fail(s, ACR_B200_JPEG_TRUNCATED); continue; }
        d.z += r;
        if (d.z > sc.se) { d.fail(s, ACR_B200_JPEG_BAD_CODE); continue; }
        if (WRITE && st->blk) st->blk[kZigzag[d.z]] = (int16_t)(extend((w << l) >> (32 - sz), sz) * (1 << sc.al));
        d.z += 1;
        d.advance(l + sz);
      } else if (r == 15) {
        d.z += 16;
        d.advance(l);
      } else if (sc.ss == 0 || r == 0) {
        d.z = 64;
        d.advance(l);
      } else {   // EOBn: this block and the next (1 << r) + bits - 1 end here
        if (l + r > avail) { d.fail(s, ACR_B200_JPEG_TRUNCATED); continue; }
        ended = (1 << r) + (int)((w << l) >> (32 - r));
        d.z = 64;
        d.advance(l + r);
      }
    }
    if (d.z > sc.se) {
      s.nblk += ended;
      if (WRITE) st->cur += ended;
      d.z = 0;
      d.c = d.c + 1 == sc.bpm ? 0 : d.c + 1;
    }
  }
}

// Last scan descriptor whose chunk_begin is <= g (unused descriptors sort after every real one).
__device__ int find_scan(const Args& a, long long g) {
  int lo = 0, hi = (int)a.max_scans - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (a.scans[mid].chunk_begin <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __maxnreg__(64) jpeg_scan_spec_kernel(Args a) {
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (g >= a.max_chunks) return;
  const acr_b200_jpeg_scan& sc = a.scans[find_scan(a, g)];
  const int j = (int)(g - sc.chunk_begin);
  if (sc.ncomp == 0 || j < 0 || j >= sc.n_chunks || sc.ah != 0 || !scan_ok(a, sc)) return;
  const acr_b200_jpeg_frame& f = a.frames[sc.frame];
  Decoder d{a.coded + sc.coded_offset, sc.coded_len, 0, 0, 0, 0, 0};
  Summary s{};
  Chunk& ch = a.chunks[g];
  if (j > 0) {
    d.guess((j - 1) * CHUNK);
    run_scan<false>(d, sc, f, j * CHUNK, s, nullptr);
    s = Summary{};
  }
  ch.from = d.state();
  run_scan<false>(d, sc, f, chunk_end(sc, j), s, nullptr);
  ch.end = d.state();
  ch.nblk = s.nblk;
  ch.dc[0] = s.dc[0], ch.dc[1] = s.dc[1], ch.dc[2] = s.dc[2];
  ch.nres = s.nres;
  ch.err = s.err;
}

struct ScanUnit {
  const Args& a;
  const acr_b200_jpeg_scan& s;
  const acr_b200_jpeg_frame& f;
  __device__ Decoder decoder() const { return Decoder{a.coded + s.coded_offset, s.coded_len, 0, 0, 0, 0, 0}; }
  __device__ void run(Decoder& d, int j, Summary& sm) const { run_scan<false>(d, s, f, chunk_end(s, j), sm, nullptr); }
};

// one CTA per scan descriptor: checks it, and synchronises a first scan's chunks
__global__ void __launch_bounds__(SYNC_THREADS, 1) jpeg_scan_sync_kernel(Args a) {
  const acr_b200_jpeg_scan& sc = a.scans[blockIdx.x];
  if (sc.ncomp == 0) return;
  if (!scan_ok(a, sc) || sc.ah != 0) {   // refinement scans are decoded by jpeg_refine_kernel
    if (threadIdx.x == 0) a.scan_status[blockIdx.x] = sc.ah != 0 && scan_ok(a, sc) ? 0 : BAD_DESC;
    return;
  }
  sync_chunks(ScanUnit{a, sc, a.frames[sc.frame]}, a.chunks + sc.chunk_begin, sc.n_chunks, sc.n_blocks,
              a.scan_status + blockIdx.x);
}

__global__ void __maxnreg__(64) jpeg_scan_write_kernel(Args a) {
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (g >= a.max_chunks) return;
  const int si = find_scan(a, g);
  const acr_b200_jpeg_scan& sc = a.scans[si];
  const int j = (int)(g - sc.chunk_begin);
  if (sc.ncomp == 0 || sc.ah != 0 || j < 0 || j >= sc.n_chunks || a.scan_status[si] != 0) return;   // status 0
                                                                                                     // implies scan_ok
  const acr_b200_jpeg_frame& f = a.frames[sc.frame];
  const Chunk& ch = a.chunks[g];
  Decoder d{a.coded + sc.coded_offset, sc.coded_len, 0, 0, 0, 0, 0};
  d.set(ch.from);
  ScanStore st{a.coef, ch.blk0, {ch.pred[0], ch.pred[1], ch.pred[2]}, nullptr};
  if (d.z > 0) st.blk = scan_block(a.coef, sc, f, st.cur);   // the chunk starts inside a block begun before it
  Summary s{};
  run_scan<true>(d, sc, f, chunk_end(sc, j), s, &st);
  if (s.err & ACR_B200_JPEG_BAD_RESTART) atomicOr(a.scan_status + si, ACR_B200_JPEG_BAD_RESTART);
}

// ---- refinement scans ------------------------------------------------------------------------------------------
// How many correction bits an AC refinement block reads depends on which of its band's coefficients are already
// nonzero, so its start cannot be guessed.  Each refinement scan runs in three steps inside one CTA:
//   masks   all threads: each block's nonzero coefficients as a 64-bit mask in zigzag order;
//   walk    one thread finds every block's start (bit position, EOB run left) from the masks alone: a block inside
//           an EOB run costs one popcount, any other block one step per code (the zero coefficients a code skips
//           are found with bit operations), and restart markers are crossed here;
//   decode  all threads, one block each from its start: the correction bits and new coefficients are stored.

// Bit reader of the refinement scans: a 64-bit buffer filled past byte stuffing, stopping at a marker.  Its whole
// state (next raw byte, buffered bits) is what the walk records for each block.
struct Bits {
  const uint8_t* seg;
  int len, b;                 // next raw byte to load
  unsigned long long buf;     // valid bits at the top
  int n;
  __device__ __forceinline__ void fill() {
    while (n <= 56 && b < len) {
      const uint32_t x = seg[b];
      if (x == 0xFF) {
        if (b + 1 < len && seg[b + 1] == 0) b += 2; else break;
      } else {
        b += 1;
      }
      buf |= (unsigned long long)x << (56 - n);
      n += 8;
    }
  }
  // k (1..32) bits, MSB first; sets err when the data ends (or a marker comes) first
  __device__ __forceinline__ uint32_t get(int k, int& err) {
    if (n < k) fill();
    if (n < k) { err |= ACR_B200_JPEG_TRUNCATED; return 0; }
    const uint32_t v = (uint32_t)(buf >> (64 - k));
    buf <<= k;
    n -= k;
    return v;
  }
  __device__ __forceinline__ void skip(int k, int& err) {
    while (k > 0 && !err) {
      const int t = min(k, 32);
      get(t, err);
      k -= t;
    }
  }
  __device__ __forceinline__ int code(const acr_b200_jpeg_huff& t, int& err) {
    if (n < 32) fill();
    int sym;
    const int l = huff(t, (uint32_t)(buf >> 32), sym);
    if (l == 0) { err |= ACR_B200_JPEG_BAD_CODE; return 0; }
    if (l > n) { err |= ACR_B200_JPEG_TRUNCATED; return 0; }
    buf <<= l;
    n -= l;
    return sym;
  }
  // Restart: drop the padding bits, then expect RSTm (after any FF fill bytes).
  __device__ int restart(int m) {
    n -= n & 7;
    if (n != 0 || b >= len || seg[b] != 0xFF) return ACR_B200_JPEG_BAD_RESTART;
    int q = b;
    while (q + 1 < len && seg[q + 1] == 0xFF) ++q;
    if (q + 1 >= len) return ACR_B200_JPEG_TRUNCATED;
    if (seg[q + 1] != 0xD0 + m) return ACR_B200_JPEG_BAD_RESTART;
    b = q + 2;
    buf = 0;
    return 0;
  }
};

// bits lo..hi (inclusive) of a 64-bit mask; empty when lo > hi
__device__ __forceinline__ unsigned long long bit_range(int lo, int hi) {
  if (lo > hi) return 0;
  const unsigned long long up = hi >= 63 ? ~0ULL : (1ULL << (hi + 1)) - 1;
  return up & ~((1ULL << lo) - 1);
}

// The walk for one AC refinement block that does not start inside an EOB run: consumes its codes and correction
// bits; returns the EOB run it leaves (0 if the block ended at Se).
__device__ __forceinline__ int walk_ac_block(Bits& d, const acr_b200_jpeg_huff& t, unsigned long long m, int ss,
                                             int se, int& err) {
  int z = ss;
  while (z <= se && !err) {
    const int sym = d.code(t, err);
    if (err) break;
    const int r = sym >> 4, s = sym & 15;
    if (s) {
      if (s != 1) { err |= ACR_B200_JPEG_BAD_CODE; break; }
      d.get(1, err);
    } else if (r != 15) {
      const int run = (1 << r) + (r ? (int)d.get(r, err) : 0);
      d.skip(__popcll(m & bit_range(z, se)), err);   // corrections of the rest of this block
      return run - 1;
    }
    // the (r+1)-th zero-history coefficient from z is the target; the nonzero ones before it get a correction bit
    unsigned long long zeros = ~m & bit_range(z, se);
    for (int q = 0; q < r && zeros; ++q) zeros &= zeros - 1;
    const int t_pos = zeros ? __ffsll((long long)zeros) - 1 : se + 1;
    d.skip(__popcll(m & bit_range(z, t_pos - 1)), err);
    if (s && t_pos > se) { err |= ACR_B200_JPEG_BAD_CODE; break; }
    z = t_pos + 1;
  }
  return 0;
}

// The decode of one refinement block from its start (libjpeg's decode_mcu_AC_refine, DC: one bit).
__device__ __forceinline__ void decode_refine_block(Bits& d, const acr_b200_jpeg_scan& sc, int16_t* blk, int c,
                                                    int eobrun, int& err) {
  const int p1 = 1 << sc.al;
  if (sc.ss == 0) {
    if (d.get(1, err)) blk[0] = (int16_t)(blk[0] | p1);
    return;
  }
  int z = sc.ss;
  if (eobrun == 0) {
    while (z <= sc.se && !err) {
      const int sym = d.code(sc.ac[c], err);
      if (err) return;
      int r = sym >> 4, val = 0;
      if (sym & 15) {
        val = d.get(1, err) ? p1 : -p1;
      } else if (r != 15) {
        if (r) d.get(r, err);
        eobrun = 1;
        break;
      }
      for (; z <= sc.se; ++z) {
        int16_t& co = blk[kZigzag[z]];
        if (co != 0) {
          if (d.get(1, err) && (co & p1) == 0) co = (int16_t)(co + (co >= 0 ? p1 : -p1));
        } else if (--r < 0) {
          break;
        }
      }
      if (val && z <= sc.se) blk[kZigzag[z]] = (int16_t)val;
      ++z;
    }
  }
  if (eobrun > 0) {
    for (; z <= sc.se; ++z) {
      int16_t& co = blk[kZigzag[z]];
      if (co != 0 && d.get(1, err) && (co & p1) == 0) co = (int16_t)(co + (co >= 0 ? p1 : -p1));
    }
  }
}

constexpr int REFINE_THREADS = 256;

// One refinement scan of frame f in the calling CTA; returns its status bits.  masks / starts: the frame's
// n_blocks-long slices of the workspace.
__device__ int refine_scan(const Args& a, const acr_b200_jpeg_scan& sc, const acr_b200_jpeg_frame& f,
                           unsigned long long* masks, int4* starts) {
  __shared__ int err_sh;
  const int tid = threadIdx.x, nb = sc.n_blocks;
  if (tid == 0) err_sh = 0;
  if (sc.ss > 0) {   // masks: zigzag order, the band only
    const unsigned long long band = bit_range(sc.ss, sc.se);
    for (int k = tid; k < nb; k += REFINE_THREADS) {
      const int16_t* blk = scan_block(a.coef, sc, f, k);
      unsigned long long m = 0;
      for (int z = sc.ss; z <= sc.se; ++z) m |= (unsigned long long)(blk[kZigzag[z]] != 0) << z;
      masks[k] = m & band;
    }
  }
  __syncthreads();
  if (tid == 0) {   // the walk
    Bits d{a.coded + sc.coded_offset, sc.coded_len, 0, 0ULL, 0};
    const int per = sc.restart * sc.bpm;
    int eobrun = 0, err = 0;
    unsigned long long next = sc.ss > 0 && nb > 0 ? masks[0] : 0;
    for (int k = 0; k < nb && !err; ++k) {
      const unsigned long long m = next;
      if (sc.ss > 0 && k + 1 < nb) next = masks[k + 1];   // the next block's mask loads while this one is walked
      if (per && k && k % per == 0) {   // the interval ends: padding, fill bytes, then the next RST
        err |= d.restart((k / per - 1) & 7);
        eobrun = 0;
        if (err) break;
      }
      starts[k] = make_int4(d.b, d.n | eobrun << 8, (int)(d.buf >> 32), (int)(uint32_t)d.buf);
      if (sc.ss == 0) {
        d.get(1, err);
      } else if (eobrun > 0) {
        d.skip(__popcll(m), err);
        --eobrun;
      } else {
        eobrun = walk_ac_block(d, sc.ac[sc.slot_comp[0]], m, sc.ss, sc.se, err);
      }
    }
    if (!err && eobrun > 0) err |= ACR_B200_JPEG_BAD_LENGTH;
    err_sh = err;
  }
  __syncthreads();
  const int walked = err_sh;
  if (walked == 0) {   // the decode
    int err = 0;
    for (int k = tid; k < nb; k += REFINE_THREADS) {
      const int4 st = starts[k];
      Bits d{a.coded + sc.coded_offset, sc.coded_len, st.x,
             (unsigned long long)(uint32_t)st.z << 32 | (uint32_t)st.w, st.y & 0xFF};
      decode_refine_block(d, sc, scan_block(a.coef, sc, f, k), sc.slot_comp[k % sc.bpm], st.y >> 8, err);
    }
    if (err) atomicOr(&err_sh, err);   // the walk read the same bits, so this never fires on data it accepted
  }
  __syncthreads();
  const int out = err_sh;
  __syncthreads();   // err_sh is reset by the next scan
  return out;
}

// Last scan descriptor whose frame is < fi, plus one: the frame's first scan.
__device__ int first_scan(const Args& a, int fi) {
  int lo = 0, hi = (int)a.max_scans;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a.scans[mid].frame < fi) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// One CTA per frame: after every first scan of the frame is in place, its refinement scans run in file order
// (refine_scan); then the frame's status, the OR of its scans'.
__global__ void __launch_bounds__(REFINE_THREADS, 1) jpeg_refine_kernel(Args a) {
  const int fi = blockIdx.x;
  const acr_b200_jpeg_frame& f = a.frames[fi];
  if (f.ncomp == 0 || f.n_scans == 0) return;
  __shared__ int first_err;
  const int tid = threadIdx.x;
  const int s0 = first_scan(a, fi);
  if (tid == 0) {
    int st = 0;
    if (!frame_geometry_ok(a, f) || s0 + (long long)f.n_scans > a.max_scans ||
        (s0 + f.n_scans < a.max_scans && a.scans[s0 + f.n_scans].frame == fi)) {
      st = BAD_DESC;
    } else {
      for (int k = 0; k < f.n_scans; ++k) st |= a.scans[s0 + k].frame == fi ? a.scan_status[s0 + k] : BAD_DESC;
    }
    first_err = st;
  }
  __syncthreads();
  int st = first_err;
  unsigned long long* masks = a.refine_masks + f.block_begin;
  int4* starts = a.refine_starts + f.block_begin;
  for (int k = 0; k < f.n_scans && st == 0; ++k) {
    const acr_b200_jpeg_scan& sc = a.scans[s0 + k];
    if (sc.ah != 0) st |= refine_scan(a, sc, f, masks, starts);
  }
  if (tid == 0) a.status[fi] = st;
}

// ---- islow IDCT: 13-bit constants, 2 pass-1 bits (Loeffler, Ligtenberg & Moschytz) -------------------------------
constexpr int CB = 13, P1 = 2;
constexpr int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
              F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

// One 8-point pass over s[0], s[step], ..., s[7 * step] in place, each result descaled by `shift` (rounded).
template <int STEP>
__device__ __forceinline__ void idct8(int* s, int shift) {
  int z2 = s[2 * STEP], z3 = s[6 * STEP];
  int z1 = (z2 + z3) * F0541;
  const int tmp2 = z1 - z3 * F1847, tmp3 = z1 + z2 * F0765;
  const int tmp0 = (s[0] + s[4 * STEP]) * (1 << CB), tmp1 = (s[0] - s[4 * STEP]) * (1 << CB);
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int a0 = s[7 * STEP], a1 = s[5 * STEP], a2 = s[3 * STEP], a3 = s[STEP];
  z1 = a0 + a3, z2 = a1 + a2, z3 = a0 + a2;
  int z4 = a1 + a3;
  const int z5 = (z3 + z4) * F1175;
  a0 *= F0298, a1 *= F2053, a2 *= F3072, a3 *= F1501;
  z1 *= -F0899, z2 *= -F2562;
  z3 = z3 * -F1961 + z5, z4 = z4 * -F0390 + z5;
  a0 += z1 + z3, a1 += z2 + z4, a2 += z2 + z3, a3 += z1 + z4;
  const int r = 1 << (shift - 1);
  s[0] = (t10 + a3 + r) >> shift, s[7 * STEP] = (t10 - a3 + r) >> shift;
  s[STEP] = (t11 + a2 + r) >> shift, s[6 * STEP] = (t11 - a2 + r) >> shift;
  s[2 * STEP] = (t12 + a1 + r) >> shift, s[5 * STEP] = (t12 - a1 + r) >> shift;
  s[3 * STEP] = (t13 + a0 + r) >> shift, s[4 * STEP] = (t13 - a0 + r) >> shift;
}

// libjpeg's post-IDCT range limit, indexed by x & 1023: -128..127 -> 0..255, 128..511 -> 255, 512..895 -> 0,
// 896..1023 -> 0..127.
__device__ __forceinline__ uint32_t range_limit(int x) {
  const int j = x & 1023;
  return j < 128 ? j + 128 : j < 512 ? 255 : j < 896 ? 0 : j - 896;
}

__global__ void __launch_bounds__(128) jpeg_idct_kernel(Args a) {
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (g >= a.max_blocks) return;
  const int fi = find_frame(a.frames, a.n, g, [](const acr_b200_jpeg_frame& f) { return (long long)f.block_begin; });
  const acr_b200_jpeg_frame& f = a.frames[fi];
  const long long l = g - f.block_begin;
  if (f.ncomp == 0 || l < 0 || l >= f.n_blocks || a.status[fi] != 0) return;
  const int c = f.ncomp == 3 && l >= f.comp_block0[2] ? 2 : f.ncomp == 3 && l >= f.comp_block0[1] ? 1 : 0;
  const int rel = (int)(l - f.comp_block0[c]), by = rel / f.comp_bw[c], bx = rel - by * f.comp_bw[c];
  int s[64];
  const int4* src = reinterpret_cast<const int4*>(a.coef + 64 * g);
  // the quantisation table is 8-byte aligned in the descriptor (offset 184, 9112-byte records): two uint2 per row
  const uint2* q = reinterpret_cast<const uint2*>(f.quant[c]);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int4 v = src[k];
    const uint2 w0 = q[2 * k], w1 = q[2 * k + 1];
    const int vv[4] = {v.x, v.y, v.z, v.w};
    const uint32_t ww[4] = {w0.x, w0.y, w1.x, w1.y};
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      s[8 * k + 2 * h] = (int)(int16_t)(vv[h] & 0xFFFF) * (int)(ww[h] & 0xFFFF);
      s[8 * k + 2 * h + 1] = (int)(int16_t)((uint32_t)vv[h] >> 16) * (int)(ww[h] >> 16);
    }
  }
#pragma unroll
  for (int col = 0; col < 8; ++col) idct8<8>(s + col, CB - P1);
  const long long stride = 8LL * f.comp_bw[c];
  uint8_t* dst = a.planes + 64 * (f.coef_offset + f.comp_block0[c]) + (8LL * by) * stride + 8 * bx;
#pragma unroll
  for (int row = 0; row < 8; ++row) {
    idct8<1>(s + 8 * row, CB + P1 + 3);
    uint2 o;
    o.x = range_limit(s[8 * row]) | range_limit(s[8 * row + 1]) << 8 | range_limit(s[8 * row + 2]) << 16 |
          range_limit(s[8 * row + 3]) << 24;
    o.y = range_limit(s[8 * row + 4]) | range_limit(s[8 * row + 5]) << 8 | range_limit(s[8 * row + 6]) << 16 |
          range_limit(s[8 * row + 7]) << 24;
    *reinterpret_cast<uint2*>(dst + row * stride) = o;
  }
}

// ---- fancy upsampling + YCbCr -> BGR ------------------------------------------------------------------------------
// Chroma sample of output pixel (x, y) for a chroma plane upsampled by (fx, fy): libjpeg-turbo's triangle filters
// (3/4 nearer + 1/4 further, alternating rounding biases), edges replicated; h2v1 / h2v2 replicate instead when the
// plane is at most 2 samples wide.
__device__ __forceinline__ int chroma(const uint8_t* p, long long stride, int cw, int ch, int fx, int fy, int x, int y) {
  if (fx == 1 && fy == 1) return p[y * stride + x];
  if (fx == 2 && cw <= 2) return p[(y / fy) * stride + (x >> 1)];
  if (fy == 1) {   // h2v1
    const int i = x >> 1, in = min(max(i + ((x & 1) ? 1 : -1), 0), cw - 1);
    const uint8_t* r = p + y * stride;
    return (3 * r[i] + r[in] + ((x & 1) ? 2 : 1)) >> 2;
  }
  const int ro = y >> 1, rn = min(max(ro + ((y & 1) ? 1 : -1), 0), ch - 1);
  const uint8_t* r0 = p + ro * stride;
  const uint8_t* r1 = p + rn * stride;
  if (fx == 1) return (3 * r0[x] + r1[x] + ((y & 1) ? 2 : 1)) >> 2;   // h1v2
  const int i = x >> 1, in = min(max(i + ((x & 1) ? 1 : -1), 0), cw - 1);   // h2v2
  const int cs = 3 * r0[i] + r1[i], cn = 3 * r0[in] + r1[in];
  return (3 * cs + cn + ((x & 1) ? 7 : 8)) >> 4;
}

__device__ __forceinline__ uint8_t clamp255(int v) { return (uint8_t)min(max(v, 0), 255); }

__global__ void __launch_bounds__(256) jpeg_color_kernel(Args a) {
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (3 * g >= a.out_bytes) return;
  const int fi = find_frame(a.frames, a.n, g, [](const acr_b200_jpeg_frame& f) { return f.out_offset / 3; });
  const acr_b200_jpeg_frame& f = a.frames[fi];
  const long long p = g - f.out_offset / 3;
  const int st = a.status[fi];
  if (f.ncomp == 0 || p < 0 || p >= (long long)f.H * f.W || (st & BAD_DESC)) return;
  if (st != 0) {   // corrupt data: a black frame, never the pixels a previous call left in the buffer
    uint8_t* o = a.out + f.out_offset + 3 * p;
    o[0] = o[1] = o[2] = 0;
    return;
  }
  const int y = (int)(p / f.W), x = (int)(p - (long long)y * f.W);
  const uint8_t* base = a.planes + 64 * f.coef_offset;
  const long long s0 = 8LL * f.comp_bw[0];
  const int Y = base[y * s0 + x];
  uint8_t* o = a.out + f.out_offset + 3 * p;
  if (f.ncomp == 1) {
    o[0] = o[1] = o[2] = (uint8_t)Y;
    return;
  }
  const int fx = f.comp_h[0], fy = f.comp_v[0];
  const int cb = chroma(base + 64LL * f.comp_block0[1], 8LL * f.comp_bw[1], f.comp_w[1], f.comp_hgt[1], fx, fy, x, y) - 128;
  const int cr = chroma(base + 64LL * f.comp_block0[2], 8LL * f.comp_bw[2], f.comp_w[2], f.comp_hgt[2], fx, fy, x, y) - 128;
  // libjpeg's tables: FIX(1.402) = 91881, FIX(1.772) = 116130, FIX(0.71414) = 46802, FIX(0.34414) = 22554 (16 bits)
  o[0] = clamp255(Y + ((116130 * cb + 32768) >> 16));
  o[1] = clamp255(Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16));
  o[2] = clamp255(Y + ((91881 * cr + 32768) >> 16));
}

size_t chunk_bytes(long long max_chunks) { return ((size_t)max_chunks * sizeof(Chunk) + 255) / 256 * 256; }

static_assert(sizeof(acr_b200_jpeg_scan) == 8632, "acr_b200_jpeg_scan layout");

}  // namespace
}  // namespace acr

using namespace acr;

extern "C" size_t acr_b200_jpeg_coef_offset(int64_t max_chunks) {
  return max_chunks < 1 ? 0 : chunk_bytes(max_chunks);
}

extern "C" size_t acr_b200_jpeg_workspace_bytes(int64_t max_chunks, int64_t max_blocks) {
  if (max_chunks < 1 || max_blocks < 1) return 0;
  return chunk_bytes(max_chunks) + (size_t)max_blocks * (128 + 64);
}

extern "C" int acr_b200_jpeg_decode(const uint8_t* coded, int64_t coded_bytes, const acr_b200_jpeg_frame* frames, int n,
                                    int64_t max_chunks, int64_t max_blocks, void* workspace, size_t workspace_bytes,
                                    uint8_t* out_bgr, int64_t out_bytes, int32_t* status, void* stream) {
  ACR_CHECK_ARG(coded && frames && workspace && out_bgr && status, "jpeg_decode: null argument");
  ACR_CHECK_ARG(n >= 1 && n <= 65535 && coded_bytes >= 0 && out_bytes >= 3 && max_chunks >= 1 &&
                    max_chunks <= 0x7fffffffLL * 128 && max_blocks >= 1 && max_blocks <= 0x7fffffffLL * 128 &&
                    out_bytes / 3 <= 0x7fffffffLL * 256,
                "jpeg_decode: bad n=%d / coded_bytes=%lld / max_chunks=%lld / max_blocks=%lld / out_bytes=%lld", n,
                (long long)coded_bytes, (long long)max_chunks, (long long)max_blocks, (long long)out_bytes);
  const size_t need = acr_b200_jpeg_workspace_bytes(max_chunks, max_blocks);
  ACR_CHECK_ARG(workspace_bytes >= need, "jpeg_decode: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  Args a{coded, (long long)coded_bytes, frames, n, (long long)max_chunks, (long long)max_blocks,
         reinterpret_cast<Chunk*>(ws), reinterpret_cast<int16_t*>(ws + chunk_bytes(max_chunks)),
         ws + chunk_bytes(max_chunks) + (size_t)max_blocks * 128, out_bgr, (long long)out_bytes, status,
         nullptr, 0, nullptr, nullptr, nullptr};
  cudaStream_t s = (cudaStream_t)stream;
  ACR_CHECK_CUDA(cudaMemsetAsync(a.coef, 0, (size_t)max_blocks * 128, s));
  const unsigned gc = (unsigned)((max_chunks + 127) / 128);
  jpeg_spec_kernel<<<gc, 128, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  jpeg_sync_kernel<<<n, SYNC_THREADS, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  jpeg_write_kernel<<<gc, 128, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  jpeg_idct_kernel<<<(unsigned)((max_blocks + 127) / 128), 128, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  jpeg_color_kernel<<<(unsigned)((out_bytes / 3 + 255) / 256), 256, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

extern "C" size_t acr_b200_jpeg_scan_workspace_bytes(int64_t max_chunks, int64_t max_blocks, int64_t max_scans) {
  if (max_chunks < 1 || max_blocks < 1 || max_scans < 1) return 0;
  return acr_b200_jpeg_workspace_bytes(max_chunks, max_blocks) + (size_t)max_blocks * 24 +
         ((size_t)max_scans * sizeof(int32_t) + 255) / 256 * 256;
}

extern "C" int acr_b200_jpeg_decode_scans(const uint8_t* coded, int64_t coded_bytes, const acr_b200_jpeg_frame* frames,
                                          int n, const acr_b200_jpeg_scan* scans, int64_t max_scans, int64_t max_chunks,
                                          int64_t max_blocks, void* workspace, size_t workspace_bytes, uint8_t* out_bgr,
                                          int64_t out_bytes, int32_t* status, void* stream) {
  ACR_CHECK_ARG(coded && frames && scans && workspace && out_bgr && status, "jpeg_decode_scans: null argument");
  ACR_CHECK_ARG(n >= 1 && n <= 65535 && coded_bytes >= 0 && out_bytes >= 3 && max_chunks >= 1 &&
                    max_chunks <= 0x7fffffffLL * 128 && max_blocks >= 1 && max_blocks <= 0x7fffffffLL * 128 &&
                    out_bytes / 3 <= 0x7fffffffLL * 256 && max_scans >= 1 && max_scans <= 65535,
                "jpeg_decode_scans: bad n=%d / coded_bytes=%lld / max_scans=%lld / max_chunks=%lld / max_blocks=%lld / "
                "out_bytes=%lld", n, (long long)coded_bytes, (long long)max_scans, (long long)max_chunks,
                (long long)max_blocks, (long long)out_bytes);
  const size_t need = acr_b200_jpeg_scan_workspace_bytes(max_chunks, max_blocks, max_scans);
  ACR_CHECK_ARG(workspace_bytes >= need, "jpeg_decode_scans: workspace of %zu bytes, %zu needed", workspace_bytes,
                need);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const size_t planes = chunk_bytes(max_chunks) + (size_t)max_blocks * 128;
  Args a{coded, (long long)coded_bytes, frames, n, (long long)max_chunks, (long long)max_blocks,
         reinterpret_cast<Chunk*>(ws), reinterpret_cast<int16_t*>(ws + chunk_bytes(max_chunks)), ws + planes, out_bgr,
         (long long)out_bytes, status, scans, (long long)max_scans,
         reinterpret_cast<int32_t*>(ws + planes + (size_t)max_blocks * 88),
         reinterpret_cast<unsigned long long*>(ws + planes + (size_t)max_blocks * 80),
         reinterpret_cast<int4*>(ws + planes + (size_t)max_blocks * 64)};   // 16-byte aligned: planes + 64 *
                                                                             // max_blocks = chunks + 192 * max_blocks
  cudaStream_t s = (cudaStream_t)stream;
  ACR_CHECK_CUDA(cudaMemsetAsync(a.coef, 0, (size_t)max_blocks * 128, s));
  const unsigned gc = (unsigned)((max_chunks + 127) / 128);
  jpeg_spec_kernel<<<gc, 128, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  jpeg_scan_spec_kernel<<<gc, 128, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  jpeg_sync_kernel<<<n, SYNC_THREADS, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  jpeg_scan_sync_kernel<<<(unsigned)max_scans, SYNC_THREADS, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  jpeg_write_kernel<<<gc, 128, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  jpeg_scan_write_kernel<<<gc, 128, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  jpeg_refine_kernel<<<n, REFINE_THREADS, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  jpeg_idct_kernel<<<(unsigned)((max_blocks + 127) / 128), 128, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  jpeg_color_kernel<<<(unsigned)((out_bytes / 3 + 255) / 256), 256, 0, s>>>(a);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}
