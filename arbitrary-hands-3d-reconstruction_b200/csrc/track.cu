// Multi-hand tracking between parse and MANO: a stable track id per detected hand and one OneEuro bank per track,
// for up to K hands per side, over B consecutive frames of one stream in one launch, or over the frames of up to S
// streams interleaved in one batch.  The statement (matching, misses, births, ids, filtering) is tests/track_ref.py,
// per stream tests/stream_track_ref.py; DESIGN.md "Multi-hand tracking" gives the reasons.
//
// One CTA per (stream, side); the state is per stream and side: a header (birth counter), K slot records (id, cell, missed, live) and K
// banks of 3 x 64 floats (previous raw value, filtered value, filtered derivative of the 45 pose values, 10 betas
// and 9 root-matrix entries: the quantities of the reference's smooth_results).  Frames go in chunks of TR_CHUNK:
//   association  warp 0 walks the row table in windows of 32 rows (coalesced), keeps a side's rows whose images
//                do not go back in time, and runs match / miss / birth per frame with the K slots in lanes 0..K-1
//                and the frame's detections in lanes 0..nd-1; the match takes the smallest packed key
//                (d2 << 8 | slot << 4 | rank) per round, a total order, with one warp min-reduction.  It writes each
//                row's id and, per frame of the chunk, the row of every slot and the births.
//   filter       thread (slot k, element e) keeps bank element e of slot k in registers and walks the chunk's
//                frames in order: the only serial recurrence.  The chunk's inputs are loaded first, all at once.
//   root         one thread per (frame, slot) turns the filtered root matrix back into an axis angle; it overlaps
//                the association of the next chunk (warp 0).
// Several streams: a one-CTA pre-pass (track_bucket_kernel) numbers the distinct streams of the batch by first frame
// and sorts the frames and the rows by (stream, side) with a stable counting sort, so the CTA of a stream walks its
// own rows only, in table order, with its frames renumbered 0..B_s-1: exactly the single-stream call on them.
// No atomics whose order reaches a result (the pre-pass's are counts and a minimum); every result is written by one
// thread in a fixed order, so repeated launches are bit-identical and one launch over B frames equals B launches of
// one frame.
#include "common.cuh"
#include "rotation.cuh"

namespace acr {

constexpr int TR_MAX_K = 16;
constexpr int TR_ELEMS = 64;          // 45 pose + 10 betas + 9 root-matrix entries
constexpr int TR_CHUNK = 8;           // frames per association / filter phase (16 spills at 64 registers)
constexpr int TR_NCELL = 64 * 64;     // flat cells of the centre map
constexpr int TR_MAX_STREAMS = 4096;  // streams of one state (the pre-pass keeps a first frame per stream in shared)
constexpr int TR_PRE_THREADS = 1024;  // the bucket pre-pass: one CTA
constexpr unsigned FULL = 0xffffffffu;

struct TrackSlot {
  int32_t id, cell, missed, live;
};

// per side: int32 births, 3 pad, TrackSlot[K], float bank[K][3][64]
__host__ __device__ constexpr size_t track_side_bytes(int K) {
  return 16 + (size_t)K * sizeof(TrackSlot) + (size_t)K * 3 * TR_ELEMS * sizeof(float);
}

// One step of the OneEuro filter (acr/utils.py:1485-1527) on one bank element:
//   x_hat = lowpass(x, alpha(mincutoff + beta*|lowpass(dx, alpha(dcutoff))|)),  dx = (x - x_prev)*freq,
//   alpha(c) = 1 / (1 + (1/(2 pi c)) / (1/freq)),  freq = 30 (te = 1/30 whatever the gap), beta = 0.7, dcutoff = 1.
__device__ __forceinline__ float one_euro_alpha(float cutoff) {
  const float te = 1.0f / 30.0f;
  const float tau = 1.0f / (2.0f * 3.14159265358979323846f * cutoff);
  return 1.0f / (1.0f + tau / te);
}

// x: the new raw value; raw, filt, fdx: the bank's previous raw value, filtered value and filtered derivative.
// Writes the filtered value xh and the filtered derivative edx.  The roundings are spelled out (which product each
// FMA absorbs), so the result does not depend on how the compiler contracts the surrounding code.
__device__ __forceinline__ void one_euro_step(float x, float mincut, float raw, float filt, float fdx, float& xh,
                                              float& edx) {
  const float dx = __fmul_rn(__fsub_rn(x, raw), 30.0f);
  const float ad = one_euro_alpha(1.0f);
  edx = __fmaf_rn(fdx, 1.0f - ad, __fmul_rn(dx, ad));
  const float a = one_euro_alpha(__fmaf_rn(fabsf(edx), 0.7f, mincut));
  xh = __fmaf_rn(a, x, __fmul_rn(1.0f - a, filt));
}

template <bool kPiTrig>
__device__ __forceinline__ float rodrigues_entry(float ax, float ay, float az, int j) {
  float R[9];
  rodrigues<kPiTrig>(ax, ay, az, R);
  float x = R[0];
#pragma unroll
  for (int i = 1; i < 9; ++i)
    if (j == i) x = R[i];
  return x;
}

// Entry j of rodrigues() in its default sincosf form.  sincosf's reduction for |angle / 2|
// >= 105615 keeps a scratch array in local memory; such angles (beyond 2e5 rad) take the sincospif form instead,
// which needs none.  The test is sincosf's own, so the compiler drops that reduction from the first branch.
__device__ __forceinline__ float track_rodrigues_entry(float ax, float ay, float az, int j) {
  const float bx = ax + 1e-8f, by = ay + 1e-8f, bz = az + 1e-8f;
  const float half = sqrtf(bx * bx + by * by + bz * bz) * 0.5f;
  return !(fabsf(half) >= 105615.0f) ? rodrigues_entry<false>(ax, ay, az, j) : rodrigues_entry<true>(ax, ay, az, j);
}

struct TrackParams {
  float* poses;
  float* betas;
  const int32_t* row_src;
  const float* flag;
  const int32_t* n_dev;
  int n_max, B, K, gate2, max_missed;
  float smooth_coeff;
  char* state;
  int32_t* track_id;
  // several streams: the pre-pass's tables (TrackWs), all nullptr for one stream's call; begin flags per frame
  const int32_t *nd, *bstream, *fr_off, *fr_list, *fr_local, *row_off, *perm;
  const int32_t* frame_begin;
};

// The pre-pass's int32 tables, in the caller's workspace: the number D of distinct streams in the batch; the stream
// of bucket j (buckets in order of first frame); per bucket its frames in batch order (fr_off / fr_list); per frame
// its index within its stream (fr_local, -1: invalid stream) and its bucket (fr_bucket); per (bucket, side) its rows
// in table order (row_off / perm).
struct TrackWs {
  int32_t *nd, *bstream, *fr_off, *fr_list, *fr_local, *fr_bucket, *row_off, *perm;
};

__host__ __device__ inline size_t track_ws_ints(int n_max, int B, int S) {
  const int P = B < S ? B : S;
  return 1 + (size_t)P + (P + 1) + 3 * (size_t)B + (2 * (size_t)P + 1) + (size_t)n_max;
}

__host__ __device__ inline TrackWs track_ws(int32_t* ws, int B, int S) {
  const int P = B < S ? B : S;
  TrackWs w;
  w.nd = ws; w.bstream = ws + 1; w.fr_off = w.bstream + P; w.fr_list = w.fr_off + P + 1; w.fr_local = w.fr_list + B;
  w.fr_bucket = w.fr_local + B; w.row_off = w.fr_bucket + B; w.perm = w.row_off + 2 * P + 1;
  return w;
}

// Exclusive scan of a[0, len) in place by the whole (TR_PRE_THREADS) CTA; out (len + 1 entries) gets the offsets and
// the total too when given.  Returns the total.
__device__ int block_scan_excl(int* a, int len, int32_t* out) {
  __shared__ int s_w[32], s_carry;
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  if (t == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < len; base += TR_PRE_THREADS) {
    const int i = base + t, v = i < len ? a[i] : 0;
    int x = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int y = __shfl_up_sync(FULL, x, off);
      if (lane >= off) x += y;
    }
    if (lane == 31) s_w[w] = x;
    __syncthreads();
    if (w == 0) {
      int y = s_w[lane];
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int z = __shfl_up_sync(FULL, y, off);
        if (lane >= off) y += z;
      }
      s_w[lane] = y;
    }
    __syncthreads();
    const int excl = s_carry + (w ? s_w[w - 1] : 0) + x - v;
    if (i < len) {
      a[i] = excl;
      if (out) out[i] = excl;
    }
    __syncthreads();
    if (t == 0) s_carry += s_w[31];
    __syncthreads();
  }
  const int total = s_carry;
  if (t == 0 && out) out[len] = total;
  __syncthreads();
  return total;
}

// Stable counting-sort scatter by the whole CTA: item i of [0, len) with key(i) >= 0 goes to position cur[key] plus
// the number of earlier items of its key (put(i, pos)), and cur advances.  Windows of TR_PRE_THREADS items; within a
// window the warps take their turns in order, each giving its lanes of one key consecutive positions.
template <class KeyF, class PutF>
__device__ void stable_scatter(int len, int* cur, KeyF key, PutF put) {
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  for (int base = 0; base < len; base += TR_PRE_THREADS) {
    const int i = base + t, k = i < len ? key(i) : -1;
    const unsigned peers = __match_any_sync(FULL, k);
    const int rank = __popc(peers & ((1u << lane) - 1u)), leader = __ffs(peers) - 1;
    for (int turn = 0; turn < TR_PRE_THREADS / 32; ++turn) {
      if (w == turn) {
        int pos = 0;
        if (lane == leader && k >= 0) {
          pos = cur[k];
          cur[k] = pos + __popc(peers);
        }
        pos = __shfl_sync(FULL, pos, leader);
        if (k >= 0) put(i, pos + rank);
      }
      __syncthreads();
    }
  }
}

struct BucketParams {
  const int32_t* row_src;
  const int32_t* n_dev;
  const int32_t* frame_stream;
  int n_max, B, S;
  int32_t* ws;
  int32_t* track_id;
};

// The pre-pass of several streams: buckets (streams in order of first frame), each frame's bucket and index within
// its stream, and the rows of each (bucket, side) in table order.  Rows that belong to no (bucket, side) -- at or past
// n_dev, image outside [0, B), a frame of an invalid stream, no side -- get id -1 here and are left untouched.
__global__ void __launch_bounds__(TR_PRE_THREADS) track_bucket_kernel(BucketParams q) {
  __shared__ int a[2 * TR_MAX_STREAMS];       // first frame per stream, then the counting sorts' cursors
  const int t = threadIdx.x, B = q.B, S = q.S;
  const TrackWs w = track_ws(q.ws, B, S);
  auto stream_of = [&](int b) { const int s = q.frame_stream[b]; return (s >= 0 && s < S) ? s : -1; };

  // 1. buckets: a frame is its stream's head when no earlier frame has that stream
  for (int s = t; s < S; s += TR_PRE_THREADS) a[s] = INT_MAX;
  __syncthreads();
  for (int b = t; b < B; b += TR_PRE_THREADS) {
    const int s = stream_of(b);
    if (s >= 0) atomicMin(&a[s], b);
  }
  __syncthreads();
  for (int b = t; b < B; b += TR_PRE_THREADS) {
    const int s = stream_of(b);
    w.fr_bucket[b] = (s >= 0 && a[s] == b) ? 1 : 0;
  }
  __syncthreads();
  const int D = block_scan_excl(w.fr_bucket, B, nullptr);    // a head's entry is now its bucket
  for (int b = t; b < B; b += TR_PRE_THREADS) {
    const int s = stream_of(b);
    if (s >= 0 && a[s] == b) w.bstream[w.fr_bucket[b]] = s;
  }
  __syncthreads();
  for (int b = t; b < B; b += TR_PRE_THREADS) {
    const int s = stream_of(b);
    if (s < 0) w.fr_bucket[b] = -1;
    else if (a[s] != b) w.fr_bucket[b] = w.fr_bucket[a[s]];    // heads keep theirs
  }
  if (t == 0) *w.nd = D;
  __syncthreads();

  // 2. each bucket's frames in batch order
  for (int j = t; j < D; j += TR_PRE_THREADS) a[j] = 0;
  __syncthreads();
  for (int b = t; b < B; b += TR_PRE_THREADS) {
    const int j = w.fr_bucket[b];
    if (j >= 0) atomicAdd(&a[j], 1);
    else w.fr_local[b] = -1;
  }
  __syncthreads();
  block_scan_excl(a, D, w.fr_off);
  stable_scatter(B, a, [&](int b) { return w.fr_bucket[b]; }, [&](int b, int pos) {
    w.fr_list[pos] = b;
    w.fr_local[b] = pos - w.fr_off[w.fr_bucket[b]];
  });

  // 3. each (bucket, side)'s rows in table order
  const int n = max(0, q.n_dev ? min(*q.n_dev, q.n_max) : q.n_max);
  auto row_key = [&](int r) {
    if (r >= n) return -1;
    const int img = q.row_src[(size_t)r * 4], side = q.row_src[(size_t)r * 4 + 1];
    if (img < 0 || img >= B || (unsigned)side > 1u) return -1;
    const int j = w.fr_bucket[img];
    return j < 0 ? -1 : 2 * j + side;
  };
  for (int j = t; j < 2 * D; j += TR_PRE_THREADS) a[j] = 0;
  __syncthreads();
  for (int r = t; r < q.n_max; r += TR_PRE_THREADS) {
    const int k = row_key(r);
    if (k >= 0) atomicAdd(&a[k], 1);
    else q.track_id[r] = -1;
  }
  __syncthreads();
  block_scan_excl(a, 2 * D, w.row_off);
  stable_scatter(q.n_max, a, row_key, [&](int r, int pos) { w.perm[pos] = r; });
}

__global__ void __launch_bounds__(TR_MAX_K * TR_ELEMS) track_kernel(TrackParams q) {
  __shared__ int s_row[2][TR_CHUNK][TR_MAX_K];     // row of slot k in frame f of the chunk, -1: none
  __shared__ unsigned s_born[2][TR_CHUNK];         // bit k: slot k's track is born in frame f
  __shared__ unsigned s_begin[2];                  // bit f: the stream starts over at frame f of the chunk
  __shared__ float s_R[TR_CHUNK][TR_MAX_K][9];     // filtered root matrices of the chunk
  const int side = blockIdx.x & 1, bucket = blockIdx.x >> 1, t = threadIdx.x, lane = t & 31, K = q.K;
  const bool smooth = q.poses != nullptr, multi = q.perm != nullptr;
  // one stream: the whole row table and B frames; several: bucket's rows [row0, row0 + n) of perm, its B frames
  // fr_list[fr0, fr0 + B) and its stream's state slot
  int B = q.B, n, row0 = 0, fr0 = 0, slot = 0;
  if (multi) {
    if (bucket >= *q.nd) return;                   // fewer distinct streams than CTAs
    fr0 = q.fr_off[bucket]; B = q.fr_off[bucket + 1] - fr0;
    row0 = q.row_off[2 * bucket + side]; n = q.row_off[2 * bucket + side + 1] - row0;
    slot = q.bstream[bucket];
  } else {
    n = max(0, q.n_dev ? min(*q.n_dev, q.n_max) : q.n_max);
  }
  char* st = q.state + ((size_t)slot * 2 + side) * track_side_bytes(K);
  int32_t* hdr = reinterpret_cast<int32_t*>(st);
  TrackSlot* slots = reinterpret_cast<TrackSlot*>(st + 16);
  float* banks = reinterpret_cast<float*>(st + 16 + (size_t)K * sizeof(TrackSlot));

  // rows of no side and rows at or past n: id -1 (the side CTAs write every other row; the pre-pass, with streams)
  if (!multi && side == 0)
    for (int r = t; r < q.n_max; r += blockDim.x)
      if (r >= n || (unsigned)q.row_src[(size_t)r * 4 + 1] > 1u) q.track_id[r] = -1;

  // ---- filter thread: bank element e of slot k
  const int k = t >> 6, e = t & 63;
  float raw = 0.f, filt = 0.f, fdx = 0.f;
  const float mincut = (e >= 45 && e < 55) ? 0.6f : q.smooth_coeff;
  if (smooth) {
    const float* bk = banks + (size_t)k * 3 * TR_ELEMS;
    raw = bk[e]; filt = bk[TR_ELEMS + e]; fdx = bk[2 * TR_ELEMS + e];
  }

  // ---- association warp: slot k in lane k, the row window in lanes
  int s_live = 0, s_id = 0, s_cell = 0, s_missed = 0, births = 0;
  int win_base = -32, w_img = 0, w_cell = 0, w_row = -1, runmax = -1;
  bool w_det = false;
  if (t < 32) {
    births = hdr[0];
    if (lane < K) {
      const TrackSlot sl = slots[lane];
      s_id = sl.id; s_cell = sl.cell; s_missed = sl.missed; s_live = sl.live != 0;
    }
  }

  // load rows [win_base, win_base + 32): a row of this side is kept when its image is in [0, B), its cell on the map
  // and its image not below any earlier kept row's (the prefix max of in-range images; an out-of-order row cannot
  // raise it); a kept row with detection_flag > 0 is a detection, every other row of this side gets id -1 here
  auto load_window = [&]() {
    const int i = win_base + lane;
    int rs = -1, img = 0, cell = 0, r = -1;
    float fl = 1.f;
    if (i < n) {
      r = multi ? q.perm[row0 + i] : i;
      const int32_t* p = q.row_src + (size_t)r * 4;
      img = p[0]; rs = p[1]; cell = p[2];
      if (multi) img = q.fr_local[img];               // the frame's index in its stream (the pre-pass checked img)
      if (q.flag) fl = q.flag[r];
    }
    const bool inr = rs == side && img >= 0 && img < B && cell >= 0 && cell < TR_NCELL;
    int v = inr ? img : -1;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int o = __shfl_up_sync(FULL, v, off);
      if (lane >= off) v = max(v, o);
    }
    int before = __shfl_up_sync(FULL, v, 1);
    if (lane == 0) before = -1;
    const bool kept = inr && img >= max(runmax, before);
    runmax = max(runmax, __shfl_sync(FULL, v, 31));
    w_det = kept && fl > 0.f;
    w_img = img; w_cell = cell; w_row = r;
    if (rs == side && !w_det) q.track_id[r] = -1;
  };

  auto associate_frame = [&](int f, int fi, int buf) {
    // 0. a begin flag: the stream's state as zeroed (a smoothing CTA's filter threads zero their banks at this frame)
    if (q.frame_begin && q.frame_begin[multi ? q.fr_list[fr0 + f] : f] != 0) {
      births = 0; s_live = 0; s_id = 0; s_cell = 0; s_missed = 0;
      if (lane == 0) s_begin[buf] |= 1u << fi;
      if (!smooth)
        for (int x = lane; x < K * 3 * TR_ELEMS; x += 32) banks[x] = 0.f;
    }
    // 1. the frame's detections, in row order, into lanes 0..nd-1 (beyond K: id -1)
    int nd = 0, d_row = -1, d_cell = 0;
    while (true) {
      const unsigned m = __ballot_sync(FULL, w_det);
      if (m == 0) {
        if (win_base + 32 >= n) break;
        win_base += 32;
        load_window();
        continue;
      }
      const int j = __ffs(m) - 1;
      if (__shfl_sync(FULL, w_img, j) != f) break;       // a later frame's
      const int cj = __shfl_sync(FULL, w_cell, j), rj = __shfl_sync(FULL, w_row, j);
      if (lane == j) w_det = false;
      if (nd < K) {
        if (lane == nd) { d_row = rj; d_cell = cj; }
        ++nd;
      } else if (lane == 0) {
        q.track_id[rj] = -1;
      }
    }
    // 2. match: pairs (slot, detection) within the gate, smallest (d2, slot, rank) first
    unsigned key[TR_MAX_K * TR_MAX_K / 32];
#pragma unroll
    for (int i = 0; i < TR_MAX_K * TR_MAX_K / 32; ++i) {
      const int p = lane + 32 * i, kk = p >> 4, d = p & 15;
      const int sc = __shfl_sync(FULL, s_cell, kk), sl = __shfl_sync(FULL, s_live, kk);
      const int dc = __shfl_sync(FULL, d_cell, d);
      const int dy = (sc >> 6) - (dc >> 6), dx = (sc & 63) - (dc & 63), d2 = dy * dy + dx * dx;
      key[i] = (kk < K && d < nd && sl && d2 <= q.gate2) ? ((unsigned)d2 << 8 | (unsigned)kk << 4 | (unsigned)d) : ~0u;
    }
    unsigned mslot = 0, mdet = 0;
    int k_det = -1, d_slot = -1;        // lane k: the detection slot k takes; lane d: the slot detection d goes to
    while (true) {
      unsigned best = ~0u;
#pragma unroll
      for (int i = 0; i < TR_MAX_K * TR_MAX_K / 32; ++i) {
        const unsigned kk = (key[i] >> 4) & 15u, d = key[i] & 15u;
        if (key[i] < best && !((mslot >> kk) & 1u) && !((mdet >> d) & 1u)) best = key[i];
      }
      best = __reduce_min_sync(FULL, best);
      if (best == ~0u) break;
      const int kk = (best >> 4) & 15, d = best & 15;
      mslot |= 1u << kk; mdet |= 1u << d;
      if (lane == kk) k_det = d;
      if (lane == d) d_slot = kk;
    }
    // 3. misses: a matched slot follows its detection, an unmatched one is freed past max_missed
    const int mcell = __shfl_sync(FULL, d_cell, k_det & 31);
    if (lane < K && s_live) {
      if ((mslot >> lane) & 1u) { s_missed = 0; s_cell = mcell; }
      else if (s_missed >= q.max_missed) s_live = 0;
      else ++s_missed;
    }
    // 4. births in row order: the lowest free slot, else the most-missed slot not matched or born in this frame
    unsigned todo = ~mdet & ((1u << nd) - 1u), bornm = 0;
    while (todo) {
      const int d = __ffs(todo) - 1;
      todo &= todo - 1;
      const int dc = __shfl_sync(FULL, d_cell, d);
      const unsigned freem = __ballot_sync(FULL, lane < K && !s_live);
      int kk;
      if (freem) {
        kk = __ffs(freem) - 1;
      } else {
        const bool cand = lane < K && !(((mslot | bornm) >> lane) & 1u);
        const int most = __reduce_max_sync(FULL, cand ? s_missed : -1);
        kk = __ffs(__ballot_sync(FULL, cand && s_missed == most)) - 1;
      }
      if (lane == kk) { s_live = 1; s_id = 2 * births + side; s_cell = dc; s_missed = 0; k_det = d; }
      if (lane == d) d_slot = kk;
      ++births;
      bornm |= 1u << kk;
    }
    // 5. outputs: the ids, and the frame's row per slot for the filter
    const int rowk = __shfl_sync(FULL, d_row, k_det & 31);
    if (lane < TR_MAX_K) s_row[buf][fi][lane] = (lane < K && k_det >= 0) ? rowk : -1;
    if (lane == 0) s_born[buf][fi] = bornm;
    const int idd = __shfl_sync(FULL, s_id, d_slot & 31);
    if (lane < nd) q.track_id[d_row] = idd;
  };

  auto associate_chunk = [&](int c) {
    const int buf = c & 1;
    if (lane == 0) s_begin[buf] = 0;
    __syncwarp();
    for (int fi = 0; fi < TR_CHUNK; ++fi) {
      const int f = c * TR_CHUNK + fi;
      if (f < B) associate_frame(f, fi, buf);
      else if (lane < TR_MAX_K) s_row[buf][fi][lane] = -1;
    }
  };

  // step c: filter chunk c - 1, then associate chunk c while the root pass finishes chunk c - 1
  const int nch = (B + TR_CHUNK - 1) / TR_CHUNK;
  for (int c = 0; c <= nch; ++c) {
    const int buf = (c - 1) & 1;
    if (smooth && c > 0) {
      // the chunk's inputs first (independent loads), then the recurrence; lanes e = 55..57 hold the root's axis
      // angle, from which every root-matrix lane of the warp computes the Rodrigues matrix
      float xs[TR_CHUNK];
#pragma unroll
      for (int fi = 0; fi < TR_CHUNK; ++fi) {
        const int r = s_row[buf][fi][k];
        xs[fi] = 0.f;
        if (r >= 0) {
          if (e < 45) xs[fi] = q.poses[(size_t)r * 48 + 3 + e];
          else if (e < 55) xs[fi] = q.betas[(size_t)r * 10 + (e - 45)];
          else if (e < 58) xs[fi] = q.poses[(size_t)r * 48 + (e - 55)];
        }
      }
#pragma unroll
      for (int fi = 0; fi < TR_CHUNK; ++fi) {
        if ((s_begin[buf] >> fi) & 1u) { raw = 0.f; filt = 0.f; fdx = 0.f; }
        const int r = s_row[buf][fi][k];                 // uniform over the slot's two warps
        if (r < 0) continue;
        float x = xs[fi];
        if (e >= 32) {
          const float ax = __shfl_sync(FULL, x, 23), ay = __shfl_sync(FULL, x, 24), az = __shfl_sync(FULL, x, 25);
          if (e >= 55) x = track_rodrigues_entry(ax, ay, az, e - 55);
        }
        float xh = x, edx = 0.f;                          // a newborn track's first frame passes through
        const bool born = (s_born[buf][fi] >> k) & 1u;
        if (!born) one_euro_step(x, mincut, raw, filt, fdx, xh, edx);
        raw = x; filt = xh; fdx = edx;
        if (e >= 55) s_R[fi][k][e - 55] = xh;
        else if (!born) {
          if (e < 45) q.poses[(size_t)r * 48 + 3 + e] = xh;
          else q.betas[(size_t)r * 10 + (e - 45)] = xh;
        }
      }
    }
    __syncthreads();
    if (t < 32) {
      if (c < nch) associate_chunk(c);
    } else if (smooth && c > 0 && t - 32 < TR_CHUNK * K) {
      const int fi = (t - 32) / K, kk = (t - 32) % K;
      const int r = s_row[buf][fi][kk];
      if (r >= 0) {
        float aa[3];
        rotmat_to_aa(&s_R[fi][kk][0], aa);
        q.poses[(size_t)r * 48 + 0] = aa[0]; q.poses[(size_t)r * 48 + 1] = aa[1]; q.poses[(size_t)r * 48 + 2] = aa[2];
      }
    }
    __syncthreads();
  }

  if (smooth) {
    float* bk = banks + (size_t)k * 3 * TR_ELEMS;
    bk[e] = raw; bk[TR_ELEMS + e] = filt; bk[2 * TR_ELEMS + e] = fdx;
  }
  if (t < 32) {
    if (lane == 0) hdr[0] = births;
    if (lane < K) {
      TrackSlot sl;
      sl.id = s_id; sl.cell = s_cell; sl.missed = s_missed; sl.live = s_live;
      slots[lane] = sl;
    }
  }
}

}  // namespace acr

using namespace acr;

extern "C" size_t acr_b200_track_state_bytes(int K) {
  return (K >= 1 && K <= TR_MAX_K) ? 2 * track_side_bytes(K) : 0;
}

extern "C" size_t acr_b200_track_streams_workspace_bytes(int n_max, int B, int S) {
  return (n_max >= 0 && B >= 1 && S >= 1 && S <= TR_MAX_STREAMS) ? track_ws_ints(n_max, B, S) * sizeof(int32_t) : 0;
}

// the checks both entry points make; fn names the entry point in the message
static int check_track_args(const char* fn, float* poses, float* betas, const int32_t* row_src, int n_max, int B, int K,
                            int gate, int max_missed, float smooth_coeff, void* state, int32_t* track_id) {
  ACR_CHECK_ARG(K >= 1 && K <= TR_MAX_K, "%s: K must be in 1..%d (got %d)", fn, TR_MAX_K, K);
  ACR_CHECK_ARG(B >= 1, "%s: B must be positive (got %d)", fn, B);
  ACR_CHECK_ARG(n_max >= 0 && (long long)n_max <= 2LL * K * B, "%s: n_max must be in 0..2*K*B = %lld (got %d)", fn,
                2LL * K * B, n_max);
  ACR_CHECK_ARG(gate >= 0 && max_missed >= 0, "%s: gate and max_missed must be >= 0 (got %d, %d)", fn, gate,
                max_missed);
  ACR_CHECK_ARG(state && row_src && track_id, "%s: null state, row table or id buffer", fn);
  ACR_CHECK_ARG((poses == nullptr) == (betas == nullptr), "%s: poses and betas must be both given or both NULL", fn);
  ACR_CHECK_ARG(poses == nullptr || smooth_coeff > 0.f, "%s: smooth_coeff must be positive when smoothing", fn);
  return ACR_B200_OK;
}

static TrackParams track_params(float* poses, float* betas, const int32_t* row_src, const float* detection_flag,
                                const int32_t* n_dev, int n_max, int B, int K, int gate, int max_missed,
                                float smooth_coeff, void* state, int32_t* track_id) {
  TrackParams q = {};
  q.poses = poses; q.betas = betas; q.row_src = row_src; q.flag = detection_flag; q.n_dev = n_dev;
  q.n_max = n_max; q.B = B; q.K = K;
  q.gate2 = min(gate, 90) * min(gate, 90);     // 63^2 + 63^2 < 90^2: a wider gate rejects nothing more
  q.max_missed = max_missed; q.smooth_coeff = smooth_coeff;
  q.state = static_cast<char*>(state); q.track_id = track_id;
  return q;
}

extern "C" int acr_b200_track_hands(float* poses, float* betas, const int32_t* row_src, const float* detection_flag,
                                    const int32_t* n_dev, int n_max, int B, int K, int gate, int max_missed,
                                    float smooth_coeff, void* state, int32_t* track_id, void* stream) {
  const int rc = check_track_args("track_hands", poses, betas, row_src, n_max, B, K, gate, max_missed, smooth_coeff,
                                  state, track_id);
  if (rc != ACR_B200_OK) return rc;
  const TrackParams q = track_params(poses, betas, row_src, detection_flag, n_dev, n_max, B, K, gate, max_missed,
                                     smooth_coeff, state, track_id);
  // ids only: the association warp alone
  track_kernel<<<2, poses ? K * TR_ELEMS : 32, 0, (cudaStream_t)stream>>>(q);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

extern "C" int acr_b200_track_streams(float* poses, float* betas, const int32_t* row_src, const float* detection_flag,
                                      const int32_t* n_dev, int n_max, int B, int K, int gate, int max_missed,
                                      float smooth_coeff, void* state, int32_t* track_id, const int32_t* frame_stream,
                                      const int32_t* frame_begin, int S, void* workspace, void* stream) {
  const int rc = check_track_args("track_streams", poses, betas, row_src, n_max, B, K, gate, max_missed, smooth_coeff,
                                  state, track_id);
  if (rc != ACR_B200_OK) return rc;
  ACR_CHECK_ARG(S >= 1 && S <= TR_MAX_STREAMS, "track_streams: S must be in 1..%d (got %d)", TR_MAX_STREAMS, S);
  ACR_CHECK_ARG(frame_stream, "track_streams: null frame_stream");
  ACR_CHECK_ARG(workspace, "track_streams: null workspace (acr_b200_track_streams_workspace_bytes)");
  BucketParams bp;
  bp.row_src = row_src; bp.n_dev = n_dev; bp.frame_stream = frame_stream;
  bp.n_max = n_max; bp.B = B; bp.S = S;
  bp.ws = static_cast<int32_t*>(workspace); bp.track_id = track_id;
  track_bucket_kernel<<<1, TR_PRE_THREADS, 0, (cudaStream_t)stream>>>(bp);
  ACR_CHECK_LAUNCH();
  TrackParams q = track_params(poses, betas, row_src, detection_flag, n_dev, n_max, B, K, gate, max_missed,
                               smooth_coeff, state, track_id);
  const TrackWs w = track_ws(bp.ws, B, S);
  q.nd = w.nd; q.bstream = w.bstream; q.fr_off = w.fr_off; q.fr_list = w.fr_list; q.fr_local = w.fr_local;
  q.row_off = w.row_off; q.perm = w.perm; q.frame_begin = frame_begin;
  // one CTA per (distinct stream, side); at most min(B, S) distinct streams, the CTAs past D return at once
  track_kernel<<<2 * min(B, S), poses ? K * TR_ELEMS : 32, 0, (cudaStream_t)stream>>>(q);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}
