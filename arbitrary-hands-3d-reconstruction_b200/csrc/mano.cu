// Fused MANO forward for sm_90a: Rodrigues -> pose/shape blend shapes -> joint regression ->
// kinematic chain -> linear blend skinning -> fingertips / joint reorder / centring ->
// weak-perspective projection, one kernel, params in -> vertices / joints out.
//
// Replaces (reference, /root/reference): ManoLayer.forward mano/manolayer.py:104-276,
// batch_rodrigues :423-434, quat2mat :396-421, MANOWrapper.forward acr/mano_wrapper.py:37-50,
// batch_orth_proj / convert_kp2d_from_input_to_orgimg acr/utils.py:384-397.
//
// Work decomposition: CTA = (group of HG hands) x (chunk of VPB vertices).  Phase 1 (all 128
// threads, thread = (hand, joint)) rebuilds the 16 rigid transforms of each hand of the group in
// shared memory -- it is ~1% of the work, so every vertex chunk recomputes it instead of taking
// a second launch or a grid sync.  Phase 2 (thread = vertex) streams the 145 blend-shape rows
// once per CTA from L2 (coalesced, [k][c][v] layout) and applies them to all HG hands from
// registers, with the pose-map coefficients broadcast from shared memory as float4.
#include "common.cuh"
#include "cam_trans.cuh"
#include "rotation.cuh"

namespace acr {

constexpr int NV = 778;
constexpr int NVP = 784;   // vertex stride in the packed model (zero padded)
constexpr int NK = 145;    // 135 pose-map rows + 10 shape rows
constexpr int HG = 8;      // hands per CTA
constexpr int VPB = 128;   // vertices per CTA == threads per CTA

constexpr size_t OFF_DIRS = 0;                              // [NK][3][NVP]
constexpr size_t OFF_VT = OFF_DIRS + (size_t)NK * 3 * NVP;  // [3][NVP]
constexpr size_t OFF_W = OFF_VT + 3 * NVP;                  // [16][NVP]
constexpr size_t OFF_JT = OFF_W + 16 * NVP;                 // [16][3]   J_regressor . v_template
constexpr size_t OFF_JS = OFF_JT + 48;                      // [16][3][10] J_regressor . shapedirs
constexpr size_t OFF_HM = OFF_JS + 480;                     // [48] 0,0,0, hands_mean
constexpr size_t MODEL_FLOATS = OFF_HM + 48;

// pose input of the layer entry points (ACR_B200_POSE_* in include/acr_b200.h)
constexpr int POSE_AXISANG = 0, POSE_ROTMAT = 1;
// root_palm: output joint 0 is the midpoint of these two vertices (manolayer.py:248-250), both in vertex chunk 0
constexpr int PALM_VA = 95, PALM_VB = 22;
static_assert(PALM_VA < VPB && PALM_VB < VPB, "the palm vertices must lie in vertex chunk 0");

// out-joint index of source joint s (inverse of the reference's reorder list, manolayer.py:254)
__constant__ int c_joint_inv[21] = {0, 5, 6, 7, 9, 10, 11, 17, 18, 19, 13, 14, 15, 1, 2, 3, 4, 8, 12, 16, 20};
// source joint of out-joint i (the reference's list itself)
__constant__ int c_joint_perm[21] = {0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20};

struct ManoParams {
  const float* model[2];  // [0]=left, [1]=right
  const float* poses;
  const float* betas;
  const int32_t* hand_type;
  int default_side;
  const int32_t* n_dev;
  int n_max;
  int center_src;  // source-joint index (0..15) used as centre, -1 none
  const float* cam;
  const float* offsets;
  float* verts;
  float* joints;
  float* center;
  float* verts_camed;
  float* pj2d;
  float* pj2d_org;
  // fused vertex all-gather (acr_b200_mano_forward_gather, protocol in include/acr_b200.h)
  int gather;                    // 0 = plain launch
  char* peer_base[8];            // every rank's symmetric allocation, mapped into this rank's address space
  char* mc_base;                 // NVLS multicast address of the same allocation, or nullptr (-> per-peer stores)
  int world, rank;
  long long dst_row;             // first row of this rank's block inside a slot (= rank * rows, even)
  unsigned long long slot_bytes, counts_offset, flags_offset;
  unsigned long long* step_dev;  // device-local: gather launches completed so far
  unsigned int* done_ctr;        // device-local: CTAs of the running launch that have finished
  const int32_t* counts_src;     // (8) int32 row counts of this shard (acr_b200_parse), carried along
};

// one value / one 16-byte vector to every GPU of the multicast group: the NVSwitch replicates the store (NVLS)
__device__ __forceinline__ void multimem_st_f32(float* mc_addr, float v) {
  asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(mc_addr), "f"(v) : "memory");
}
__device__ __forceinline__ void multimem_st_v4(float* mc_addr, const float4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// bounded spin on arrival flags in THIS rank's memory: a peer that never arrives must fail the launch, not hang the box
__device__ __forceinline__ void wait_flag_ge(const unsigned long long* flag, unsigned long long target) {
  const long long t0 = clock64();
  while (ld_acquire_sys(flag) < target) {
    __nanosleep(200);
    if (clock64() - t0 > 60000000000ll) {   // ~30 s
      printf("acr_b200 gather: rank flag %p stuck at %llu < %llu\n", (const void*)flag, ld_acquire_sys(flag), target);
      __trap();
    }
  }
}

// fp32 pairs kept in one 64-bit value; Hopper has no packed fp32 FMA, so each lane is one plain IEEE fmaf
// (results are bit-identical to a scalar loop)
__device__ __forceinline__ unsigned long long pk2(float lo, float hi) {
  unsigned long long r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void ffma2(unsigned long long& acc, unsigned long long a, unsigned long long b) {
  asm("{\n.reg .f32 a0, a1, b0, b1, c0, c1;\n"
      "mov.b64 {a0, a1}, %1;\nmov.b64 {b0, b1}, %2;\nmov.b64 {c0, c1}, %0;\n"
      "fma.rn.f32 c0, a0, b0, c0;\nfma.rn.f32 c1, a1, b1, c1;\nmov.b64 %0, {c0, c1};\n}"
      : "+l"(acc) : "l"(a), "l"(b));
}
__device__ __forceinline__ void unpk2(unsigned long long v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}

constexpr int STAGE_ROW = 4 + VPB * 3;   // floats: a hand's 384 vertex floats at the offset that matches their global alignment

struct ProjCtx {  // per-hand projection constants kept in shared memory
  float s, tx, ty, padw, padh, ltx, lty;
};

__device__ __forceinline__ void write_joint(const ManoParams& p, int hand, int out_idx, float x, float y,
                                            float z, const ProjCtx& pc) {
  if (p.joints) {
    float* o = p.joints + ((size_t)hand * 21 + out_idx) * 3;
    o[0] = x; o[1] = y; o[2] = z;
  }
  if (p.cam) {
    float px = x * pc.s + pc.tx, py = y * pc.s + pc.ty;
    if (p.pj2d) {
      float* o = p.pj2d + ((size_t)hand * 21 + out_idx) * 2;
      o[0] = px; o[1] = py;
    }
    if (p.pj2d_org && p.offsets) {
      float* o = p.pj2d_org + ((size_t)hand * 21 + out_idx) * 2;
      o[0] = (px + 1.f) * pc.padw / 2.f + pc.ltx;
      o[1] = (py + 1.f) * pc.padh / 2.f + pc.lty;
    }
  }
}

// Phase 1, shared by the forward and both backward kernels: thread (h, j) of a 128-thread CTA rebuilds joint j of
// hand h of the group -- its Rodrigues rotation, rest joint and pose-map rows -- then threads j<5 walk the five
// fingers (three levels each), and every thread forms its skinning transform A_j.  `m` is the packed model of the
// hand; a row beyond n (!valid, m unused) gets the identity rotation, a zero joint and zero blend coefficients.
// Ends synchronised.  kPiTrig as in rodrigues(): the backward kernels use it, so they never touch local memory.
// kPose: POSE_AXISANG reads (n,48) axis angles (the mean pose is added here); POSE_ROTMAT reads (n,16,3,3) matrices
// and projects each onto SO(3) like the reference's batch_rotprojs (no mean pose: its rotmat branch has none).
template <bool kPiTrig = false, int kPose = POSE_AXISANG>
__device__ __forceinline__ void rebuild_transforms(bool valid, const float* __restrict__ m, const float* __restrict__ poses,
                                                   const float* __restrict__ betas, int hand, int h, int j, int center_src,
                                                   float (*s_pm)[HG], float (*s_A)[16][12], float (*s_R)[16][9],
                                                   float (*s_J)[16][3], float (*s_G)[16][12], float (*s_ctr)[3]) {
  float R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  float J[3] = {0, 0, 0};
  if (valid) {
    if constexpr (kPose == POSE_ROTMAT) {
      so3_project(poses + ((size_t)hand * 16 + j) * 9, R);
    } else {
      const float* ps = poses + (size_t)hand * 48 + j * 3;
      float ax = ps[0] + m[OFF_HM + j * 3 + 0];
      float ay = ps[1] + m[OFF_HM + j * 3 + 1];
      float az = ps[2] + m[OFF_HM + j * 3 + 2];
      rodrigues<kPiTrig>(ax, ay, az, R);
    }
    const float* b = betas + (size_t)hand * 10;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float a = m[OFF_JT + j * 3 + c];
      const float* js = m + OFF_JS + (j * 3 + c) * 10;
#pragma unroll
      for (int k = 0; k < 10; ++k) a = fmaf(js[k], b[k], a);
      J[c] = a;
    }
    if (j < 10) s_pm[135 + j][h] = b[j];
  } else if (j < 10) {
    s_pm[135 + j][h] = 0.f;
  }
#pragma unroll
  for (int e = 0; e < 9; ++e) s_R[h][j][e] = R[e];
#pragma unroll
  for (int c = 0; c < 3; ++c) s_J[h][j][c] = J[c];
  if (j >= 1) {
#pragma unroll
    for (int e = 0; e < 9; ++e) s_pm[(j - 1) * 9 + e][h] = valid ? R[e] - ((e & 3) == 0 ? 1.f : 0.f) : 0.f;
  }
  __syncthreads();
  // kinematic chain: thread j<5 walks finger j (joints 3j+1..3j+3); thread j==5 stores the root
  if (j <= 5) {
    float G[12];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      G[r * 4 + 0] = s_R[h][0][r * 3 + 0]; G[r * 4 + 1] = s_R[h][0][r * 3 + 1];
      G[r * 4 + 2] = s_R[h][0][r * 3 + 2]; G[r * 4 + 3] = s_J[h][0][r];
    }
    if (j == 5) {
#pragma unroll
      for (int e = 0; e < 12; ++e) s_G[h][0][e] = G[e];
    } else {
      int parent = 0;
#pragma unroll
      for (int lev = 0; lev < 3; ++lev) {
        const int idx = 3 * j + 1 + lev;
        const float* Rl = s_R[h][idx];
        float rel[3] = {s_J[h][idx][0] - s_J[h][parent][0], s_J[h][idx][1] - s_J[h][parent][1],
                        s_J[h][idx][2] - s_J[h][parent][2]};
        float N[12];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
#pragma unroll
          for (int c = 0; c < 3; ++c)
            N[r * 4 + c] = G[r * 4 + 0] * Rl[0 * 3 + c] + G[r * 4 + 1] * Rl[1 * 3 + c] + G[r * 4 + 2] * Rl[2 * 3 + c];
          N[r * 4 + 3] = G[r * 4 + 0] * rel[0] + G[r * 4 + 1] * rel[1] + G[r * 4 + 2] * rel[2] + G[r * 4 + 3];
        }
#pragma unroll
        for (int e = 0; e < 12; ++e) { G[e] = N[e]; s_G[h][idx][e] = N[e]; }
        parent = idx;
      }
    }
  }
  __syncthreads();
  // A_j = [R_g | t_g - R_g . J_j]   (manolayer.py:226-228)
  {
    const float* G = s_G[h][j];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      s_A[h][j][r * 4 + 0] = G[r * 4 + 0]; s_A[h][j][r * 4 + 1] = G[r * 4 + 1]; s_A[h][j][r * 4 + 2] = G[r * 4 + 2];
      s_A[h][j][r * 4 + 3] = G[r * 4 + 3] - (G[r * 4 + 0] * J[0] + G[r * 4 + 1] * J[1] + G[r * 4 + 2] * J[2]);
    }
  }
  if (j < 3) s_ctr[h][j] = (center_src >= 0) ? s_G[h][center_src][j * 4 + 3] : 0.f;
  __syncthreads();
}

// v_posed of vertex column vc for the HG hands of the group: template + 145 blend rows (streamed from L2, coalesced
// [k][c][v] layout) times the per-hand coefficients broadcast from shared memory.
__device__ __forceinline__ void blend_vertex(const float* __restrict__ m, int vc, const float (*s_pm)[HG], float (&acc)[HG][3]) {
  const float* __restrict__ dirs = m + OFF_DIRS;
  unsigned long long acc2[HG / 2][3];   // (hand 2i, hand 2i+1) packed: one ffma2 (two fp32 FMAs) serves two hands
  {
    const float v0 = m[OFF_VT + 0 * NVP + vc], v1 = m[OFF_VT + 1 * NVP + vc], v2 = m[OFF_VT + 2 * NVP + vc];
#pragma unroll
    for (int h = 0; h < HG / 2; ++h) { acc2[h][0] = pk2(v0, v0); acc2[h][1] = pk2(v1, v1); acc2[h][2] = pk2(v2, v2); }
  }
  // shape rows first (v_shaped), then pose rows, like the reference's evaluation order
#pragma unroll 5
  for (int kk = 0; kk < NK; ++kk) {
    const int k = (kk < 10) ? 135 + kk : kk - 10;
    const float d0 = __ldg(dirs + ((size_t)k * 3 + 0) * NVP + vc);
    const float d1 = __ldg(dirs + ((size_t)k * 3 + 1) * NVP + vc);
    const float d2 = __ldg(dirs + ((size_t)k * 3 + 2) * NVP + vc);
    const float4 pa = *reinterpret_cast<const float4*>(&s_pm[k][0]);
    const float4 pb = *reinterpret_cast<const float4*>(&s_pm[k][4]);
    const unsigned long long D0 = pk2(d0, d0), D1 = pk2(d1, d1), D2 = pk2(d2, d2);
    const unsigned long long P[4] = {pk2(pa.x, pa.y), pk2(pa.z, pa.w), pk2(pb.x, pb.y), pk2(pb.z, pb.w)};
#pragma unroll
    for (int h = 0; h < HG / 2; ++h) {
      ffma2(acc2[h][0], D0, P[h]);
      ffma2(acc2[h][1], D1, P[h]);
      ffma2(acc2[h][2], D2, P[h]);
    }
  }
#pragma unroll
  for (int h = 0; h < HG / 2; ++h)
#pragma unroll
    for (int c = 0; c < 3; ++c) unpk2(acc2[h][c], acc[2 * h][c], acc[2 * h + 1][c]);
}

// skinning transform of one vertex: T = sum_j w_j A_j (3x4, row-major)
__device__ __forceinline__ void skin_transform(const float (&w)[16], const float (*A)[12], float (&T)[12]) {
#pragma unroll
  for (int e = 0; e < 12; ++e) T[e] = 0.f;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float4 a0 = *reinterpret_cast<const float4*>(&A[j][0]);
    const float4 a1 = *reinterpret_cast<const float4*>(&A[j][4]);
    const float4 a2 = *reinterpret_cast<const float4*>(&A[j][8]);
    T[0] = fmaf(w[j], a0.x, T[0]); T[1] = fmaf(w[j], a0.y, T[1]); T[2] = fmaf(w[j], a0.z, T[2]); T[3] = fmaf(w[j], a0.w, T[3]);
    T[4] = fmaf(w[j], a1.x, T[4]); T[5] = fmaf(w[j], a1.y, T[5]); T[6] = fmaf(w[j], a1.z, T[6]); T[7] = fmaf(w[j], a1.w, T[7]);
    T[8] = fmaf(w[j], a2.x, T[8]); T[9] = fmaf(w[j], a2.y, T[9]); T[10] = fmaf(w[j], a2.z, T[10]); T[11] = fmaf(w[j], a2.w, T[11]);
  }
}

// The forward, for the pose input kPose; kPalm replaces output joint 0 (the wrist) by the palm, the midpoint of
// vertices 95 and 22, which the chunk-0 CTA takes from its staged vertices.
template <int kPose, bool kPalm>
__device__ __forceinline__ void mano_forward_body(const ManoParams p) {
  constexpr bool kGather = kPose == POSE_AXISANG && !kPalm;   // the fused all-gather is compiled into this form only
  __shared__ __align__(16) float s_pm[NK][HG];        // pose-map / beta coefficients, [k][hand]
  __shared__ __align__(16) float s_A[HG][16][12];     // skinning transforms (rest pose removed)
  __shared__ float s_R[HG][16][9];                    // local rotations
  __shared__ float s_J[HG][16][3];                    // rest joints
  __shared__ float s_G[HG][16][12];                   // global transforms
  __shared__ float s_ctr[HG][3];
  __shared__ ProjCtx s_pc[HG];
  __shared__ int s_side[HG];
  __shared__ __align__(16) float s_stage[HG][STAGE_ROW];   // vertices of this CTA, staged for 16-byte stores
  __shared__ int s_last;

  const int n = p.n_dev ? min(*p.n_dev, p.n_max) : p.n_max;
  const int g0 = blockIdx.x * HG;
  const int t = threadIdx.x;
  // ---- fused all-gather bookkeeping.  This launch is gather step `step + 1`; it writes slot (step + 1) & 1.
  unsigned long long step = 0;
  char* slot_mc = nullptr;
  unsigned long long slot_off = 0;
  if (kGather && p.gather) {
    step = *p.step_dev;                       // stable during the launch: only the last CTA advances it, at the very end
    slot_off = ((step + 1) & 1ull) * p.slot_bytes;
    slot_mc = p.mc_base ? p.mc_base + slot_off : nullptr;
    // CTA (0,0) carries the 32 bytes of row counts of this shard to every rank (no separate collective)
    if (blockIdx.x == 0 && blockIdx.y == 0 && t < 8 && p.counts_src) {
      // the slot is free once every peer has signalled step `step` (see below)
      for (int r = 0; r < p.world; ++r) wait_flag_ge(reinterpret_cast<const unsigned long long*>(p.peer_base[p.rank] + p.flags_offset) + r, step);
      const int32_t cv = p.counts_src[t];
      const unsigned long long off = slot_off + p.counts_offset + ((size_t)p.rank * 8 + t) * 4;
      if (p.mc_base) multimem_st_f32(reinterpret_cast<float*>(p.mc_base + off), __int_as_float(cv));
      else for (int r = 0; r < p.world; ++r) *reinterpret_cast<int32_t*>(p.peer_base[r] + off) = cv;
    }
  }
  const bool active = g0 < n;
  if (active && kGather && p.gather) {
    // Slot (step+1)&1 was last written by step-1.  A peer signals step `step` only after its launch `step`, which it
    // enqueued after consuming step-1's data (the consume-before-next-launch contract) -> once every peer's flag in
    // OUR memory reads >= step, nobody reads the slot any more.  With two slots this wait is one whole step old.
    if (t < p.world) wait_flag_ge(reinterpret_cast<const unsigned long long*>(p.peer_base[p.rank] + p.flags_offset) + t, step);
    __syncthreads();
  }
  if (active) {

  // ---------------------------------------------------------------- phase 1: rigid transforms
  {
    const int h = t >> 4, j = t & 15;
    const int hand = g0 + h;
    const bool valid = hand < n;
    int side = p.default_side;
    if (valid && p.hand_type) side = p.hand_type[hand] != 0;
    if (!valid) side = -1;
    if (j == 0) {
      s_side[h] = side;
      ProjCtx pc = {1.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (valid && p.cam) {
        pc.s = p.cam[hand * 3 + 0]; pc.tx = p.cam[hand * 3 + 1]; pc.ty = p.cam[hand * 3 + 2];
        if (p.offsets) {  // [pad_h,pad_w | crop t,r,b,l | pad t,r,b,l]  (acr/utils.py:392-397)
          const float* o = p.offsets + (size_t)hand * 10;
          pc.padw = o[0]; pc.padh = o[1];  // kp2d.x scales with offsets[:,0], kp2d.y with [:,1]
          pc.ltx = o[5] - o[9];
          pc.lty = o[2] - o[6];
        }
      }
      s_pc[h] = pc;
    }
    rebuild_transforms<false, kPose>(valid, p.model[valid ? side : 0], p.poses, p.betas, hand, h, j, p.center_src, s_pm,
                                     s_A, s_R, s_J, s_G, s_ctr);
    // kinematic joints + centre are written once per hand group (vertex chunk 0)
    if (blockIdx.y == 0 && valid) {
      const float* G = s_G[h][j];
      if (!(kPalm && j == 0))
        write_joint(p, hand, c_joint_inv[j], G[3] - s_ctr[h][0], G[7] - s_ctr[h][1], G[11] - s_ctr[h][2], s_pc[h]);
      if (j < 3 && p.center) p.center[(size_t)hand * 3 + j] = s_ctr[h][j];
    }
  }

  // ------------------------------------------------------------------ phase 2: vertices
  const int v = blockIdx.y * VPB + t;
  const bool vvalid = v < NV;
  const int vc = vvalid ? v : NVP - 1;  // padded (zero) column for the idle tail threads
  for (int side = 0; side < 2; ++side) {
    bool any = false;
#pragma unroll
    for (int h = 0; h < HG; ++h) any |= (s_side[h] == side);
    if (!any) continue;  // block-uniform
    const float* __restrict__ m = p.model[side];
    float acc[HG][3];
    blend_vertex(m, vc, s_pm, acc);
    float w[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) w[j] = __ldg(m + OFF_W + j * NVP + vc);
    // fingertip slot of this vertex (manolayer.py:244-247), -1 if none
    int tip = -1;
    if (v == 745) tip = 0; else if (v == 317) tip = 1; else if (v == (side ? 444 : 445)) tip = 2;
    else if (v == 556) tip = 3; else if (v == 673) tip = 4;
#pragma unroll
    for (int h = 0; h < HG; ++h) {
      if (s_side[h] != side) continue;  // block-uniform
      float T[12];
      skin_transform(w, s_A[h], T);
      const float x = T[0] * acc[h][0] + T[1] * acc[h][1] + T[2] * acc[h][2] + T[3] - s_ctr[h][0];
      const float y = T[4] * acc[h][0] + T[5] * acc[h][1] + T[6] * acc[h][2] + T[7] - s_ctr[h][1];
      const float z = T[8] * acc[h][0] + T[9] * acc[h][1] + T[10] * acc[h][2] + T[11] - s_ctr[h][2];
      if (!vvalid) continue;
      const int hand = g0 + h;
      {   // stage at the offset that matches the global alignment of this hand's chunk (phase 3)
        const int o = (int)((((size_t)hand * NV + (size_t)blockIdx.y * VPB) * 3) & 3);
        float* sp = &s_stage[h][o + 3 * t];
        sp[0] = x; sp[1] = y; sp[2] = z;
      }
      if (tip >= 0) write_joint(p, hand, c_joint_inv[16 + tip], x, y, z, s_pc[h]);
    }
  }

  // ---------------------------------------------------------------- phase 3: 16-byte vertex stores
  // A hand's chunk is 3*nv contiguous floats at global float index gidx = (hand*778 + v0)*3, which is 8-byte but
  // not always 16-byte aligned (778*3 = 2 mod 4).  It was staged at offset (gidx & 3) of its shared-memory row, so
  // 16-byte chunk j of the row IS an aligned 16-byte chunk of global memory: one float4 (or multimem.st.v4 / peer
  // float4) per thread and chunk; the first / last chunk of a row may be partial and falls back to scalar stores.
  __syncthreads();
  if constexpr (kPalm) {   // palm = (v95 + v22) / 2 of the (centred) staged vertices, in place of the wrist
    if (blockIdx.y == 0 && t < HG && s_side[t] >= 0) {
      const int hand = g0 + t;
      const float* sp = &s_stage[t][(int)(((size_t)hand * NV * 3) & 3)];
      write_joint(p, hand, 0, (sp[3 * PALM_VA + 0] + sp[3 * PALM_VB + 0]) * 0.5f,
                  (sp[3 * PALM_VA + 1] + sp[3 * PALM_VB + 1]) * 0.5f, (sp[3 * PALM_VA + 2] + sp[3 * PALM_VB + 2]) * 0.5f,
                  s_pc[t]);
    }
  }
  {
    const int v0 = blockIdx.y * VPB;
    const int nfl = min(VPB, NV - v0) * 3;
    for (int h = 0; h < HG; ++h) {
      if (s_side[h] < 0) continue;                      // block-uniform
      const int hand = g0 + h;
      const size_t gidx = ((size_t)hand * NV + v0) * 3;
      const int o = (int)(gidx & 3);
      const size_t gg = ((size_t)(p.dst_row + hand) * NV + v0) * 3;      // same (gg & 3): dst_row is even
      const int nchunk = (o + nfl + 3) >> 2;
      const float sc = s_pc[h].s, tx = s_pc[h].tx, ty = s_pc[h].ty;
      for (int j = t; j < nchunk; j += VPB) {
        const float4 q = *reinterpret_cast<const float4*>(&s_stage[h][4 * j]);
        const float e[4] = {q.x, q.y, q.z, q.w};
        const int i0 = 4 * j - o;                       // float index inside the chunk of element 0 (may be < 0)
        const bool full = i0 >= 0 && i0 + 4 <= nfl;
        float c4[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int comp = (i0 + k + 3) % 3;            // i0 + k >= -3
          c4[k] = comp == 0 ? e[k] * sc + tx : (comp == 1 ? e[k] * sc + ty : e[k]);
        }
        if (full) {
          if (p.verts) *reinterpret_cast<float4*>(p.verts + gidx + i0) = q;
          if (p.verts_camed && p.cam) *reinterpret_cast<float4*>(p.verts_camed + gidx + i0) = make_float4(c4[0], c4[1], c4[2], c4[3]);
          if (kGather && p.gather) {
            const unsigned long long off = slot_off + (gg + i0) * 4;
            if (slot_mc) multimem_st_v4(reinterpret_cast<float*>(p.mc_base + off), q);
            else for (int r = 0; r < p.world; ++r) *reinterpret_cast<float4*>(p.peer_base[r] + off) = q;
          }
        } else {
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int i = i0 + k;
            if (i < 0 || i >= nfl) continue;
            if (p.verts) p.verts[gidx + i] = e[k];
            if (p.verts_camed && p.cam) p.verts_camed[gidx + i] = c4[k];
            if (kGather && p.gather) {
              const unsigned long long off = slot_off + (gg + i) * 4;
              if (slot_mc) multimem_st_f32(reinterpret_cast<float*>(p.mc_base + off), e[k]);
              else for (int r = 0; r < p.world; ++r) *reinterpret_cast<float*>(p.peer_base[r] + off) = e[k];
            }
          }
        }
      }
    }
  }
  }  // if (active)

  // ---------------------------------------------------------------- gather: completion signal
  // Every CTA (also the ones beyond n) counts itself done after a system-scope fence; the last one to finish
  // publishes step+1 in the flag word flags[rank] of EVERY rank (release, system scope): whoever acquires that
  // value sees all vertices and counts of this launch.  No separate barrier kernel, no NCCL call.
  if (kGather && p.gather) {
    __syncthreads();
    if (t == 0) {
      __threadfence_system();
      const unsigned int total = gridDim.x * gridDim.y;
      s_last = (atomicAdd(p.done_ctr, 1u) == total - 1) ? 1 : 0;
    }
    __syncthreads();
    if (s_last) {
      if (t == 0) { __threadfence_system(); *p.done_ctr = 0u; }
      __syncthreads();
      if (t < p.world)
        st_release_sys(reinterpret_cast<unsigned long long*>(p.peer_base[t] + p.flags_offset) + p.rank, step + 1);
      if (t == 0) *p.step_dev = step + 1;
    }
  }
}

__global__ void __launch_bounds__(VPB) mano_forward_kernel(const ManoParams p) { mano_forward_body<POSE_AXISANG, false>(p); }

// the other forms of acr_b200_mano_layer_forward (axis angle without the palm is mano_forward_kernel itself)
template <int kPose, bool kPalm>
__global__ void __launch_bounds__(VPB) mano_layer_forward_kernel(const ManoParams p) { mano_forward_body<kPose, kPalm>(p); }

// stream-ordered wait until the stores of the most recent gather launch of EVERY rank have landed in this rank's memory
__global__ void gather_wait_kernel(const unsigned long long* flags, const unsigned long long* step_dev, int world) {
  if ((int)threadIdx.x < world) wait_flag_ge(flags + threadIdx.x, *step_dev);
}

// estimate_translation_np for one hand per thread (cam_trans.cuh)
__global__ void cam_trans_kernel(const float* __restrict__ j3d, const float* __restrict__ pj2d,
                                 const int32_t* __restrict__ n_dev, int n_max, float focal, float img_size,
                                 float* __restrict__ out) {
  const int n = n_dev ? min(*n_dev, n_max) : n_max;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  cam_trans_lstsq(j3d + (size_t)i * 63, pj2d + (size_t)i * 42, focal, img_size, out + (size_t)i * 3);
}

__global__ void rodrigues_kernel(const float* __restrict__ aa, int n, float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float R[9];
  rodrigues(aa[i * 3 + 0], aa[i * 3 + 1], aa[i * 3 + 2], R);
#pragma unroll
  for (int e = 0; e < 9; ++e) out[(size_t)i * 9 + e] = R[e];
}

__global__ void rot6d_to_aa_kernel(const float* __restrict__ r6, int n, float* __restrict__ aa) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float o[3];
  rot6d_to_aa(r6 + (size_t)i * 6, o);
  aa[i * 3 + 0] = o[0]; aa[i * 3 + 1] = o[1]; aa[i * 3 + 2] = o[2];
}

// ------------------------------------------------------------------------------------------------- MANO backward
// Two launches, no atomics, nothing saved from the forward.
//   vertex kernel (forward grid): rebuild phase 1, recompute v_posed and the skinning transform T of every vertex,
//     take its cotangent du (dverts + the joint cotangent of a fingertip) and reduce, per CTA and hand,
//       dA_j = sum_v w_vj [du v_posed^T | du]        (16 x 3x4)
//       dpm_k = sum_v dirs_k . (T[:, :3]^T du)       (145 blend-row coefficients)
//       sum_v du                                     (for the centre)
//     into the caller's workspace, one fixed-order partial per (hand, vertex chunk).
//   chain kernel (one CTA per HG hands, thread = (hand, joint)): sum the partials over the chunks in order, run the
//     A_j and chain backward (tips to root), Rodrigues backward, and the J_regressor . shapedirs term of dbetas.
constexpr int NCHUNK = (NV + VPB - 1) / VPB;   // vertex chunks per hand
constexpr int WS_DA = 0, WS_DPM = 192, WS_DU = WS_DPM + NK, WS_STRIDE = WS_DU + 3;   // floats per (hand, chunk)
constexpr int DUVP_STRIDE = VPB * 6 + 2;       // per hand: (du, v_posed) of every vertex; +2 spreads the banks

struct ManoGradParams {
  const float* model;
  int side;
  const float* poses;
  const float* betas;
  int n;
  int center_src;
  const float* dverts;
  const float* djoints;
  const float* dcenter;
  float* ws;
  int have_partials;   // 0: no vertex / joint cotangent, the vertex kernel did not run
  float* dposes;
  float* dbetas;
};

constexpr size_t GRAD_DYN_SMEM = (size_t)(HG * DUVP_STRIDE + 3 * VPB * HG + 3 * NK * HG) * sizeof(float);

// kPose / kPalm as in mano_forward_body: with the palm, half of output joint 0's cotangent joins the du of each of
// vertices 95 and 22.
template <int kPose, bool kPalm>
__device__ __forceinline__ void mano_backward_vertex_body(const ManoGradParams p) {
  __shared__ __align__(16) float s_pm[NK][HG];
  __shared__ __align__(16) float s_A[HG][16][12];
  __shared__ float s_R[HG][16][9];
  __shared__ float s_J[HG][16][3];
  __shared__ float s_G[HG][16][12];
  __shared__ float s_ctr[HG][3];
  extern __shared__ __align__(16) float s_dyn[];
  float* s_duvp = s_dyn;                        // [HG][DUVP_STRIDE]
  float* s_dvp = s_duvp + HG * DUVP_STRIDE;     // [3][VPB][HG]   d v_posed
  float* s_dpm3 = s_dvp + 3 * VPB * HG;         // [3][NK][HG]    dpm per coordinate

  const int g0 = blockIdx.x * HG;
  const int t = threadIdx.x;
  const float* __restrict__ m = p.model;
  {
    const int h = t >> 4, j = t & 15;
    rebuild_transforms<true, kPose>(g0 + h < p.n, m, p.poses, p.betas, g0 + h, h, j, p.center_src, s_pm, s_A, s_R, s_J,
                                    s_G, s_ctr);
  }
  const int v0 = blockIdx.y * VPB;
  const int nv = min(VPB, NV - v0);
  // ---- per vertex: du, v_posed and d v_posed = T[:, :3]^T du of every hand
  {
    const int v = v0 + t;
    const bool vvalid = v < NV;
    const int vc = vvalid ? v : NVP - 1;
    float acc[HG][3];
    blend_vertex(m, vc, s_pm, acc);
    float w[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) w[j] = __ldg(m + OFF_W + j * NVP + vc);
    int tip = -1;
    if (v == 745) tip = 0; else if (v == 317) tip = 1; else if (v == (p.side ? 444 : 445)) tip = 2;
    else if (v == 556) tip = 3; else if (v == 673) tip = 4;
#pragma unroll
    for (int h = 0; h < HG; ++h) {
      const int hand = g0 + h;
      float du[3] = {0.f, 0.f, 0.f};
      if (vvalid && hand < p.n) {
        if (p.dverts) {
          const float* d = p.dverts + ((size_t)hand * NV + v) * 3;
          du[0] = d[0]; du[1] = d[1]; du[2] = d[2];
        }
        if (tip >= 0 && p.djoints) {
          const float* d = p.djoints + ((size_t)hand * 21 + c_joint_inv[16 + tip]) * 3;
          du[0] += d[0]; du[1] += d[1]; du[2] += d[2];
        }
        if (kPalm && (v == PALM_VA || v == PALM_VB) && p.djoints) {
          const float* d = p.djoints + (size_t)hand * 21 * 3;
          du[0] += 0.5f * d[0]; du[1] += 0.5f * d[1]; du[2] += 0.5f * d[2];
        }
      }
      float T[12];
      skin_transform(w, s_A[h], T);
      float* o = s_duvp + h * DUVP_STRIDE + t * 6;
      o[0] = du[0]; o[1] = du[1]; o[2] = du[2]; o[3] = acc[h][0]; o[4] = acc[h][1]; o[5] = acc[h][2];
#pragma unroll
      for (int c = 0; c < 3; ++c)
        s_dvp[(c * VPB + t) * HG + h] = T[0 * 4 + c] * du[0] + T[1 * 4 + c] * du[1] + T[2 * 4 + c] * du[2];
    }
  }
  __syncthreads();
  // ---- dA_j and sum(du): thread (h, j), vertices in order
  {
    const int h = t >> 4, j = t & 15;
    const float* __restrict__ wj = m + OFF_W + (size_t)j * NVP + v0;
    const float* d = s_duvp + h * DUVP_STRIDE;
    float a[12], su[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int e = 0; e < 12; ++e) a[e] = 0.f;
    for (int i = 0; i < nv; ++i) {
      const float wv = __ldg(wj + i);
      const float2 q0 = *reinterpret_cast<const float2*>(d + 6 * i);
      const float2 q1 = *reinterpret_cast<const float2*>(d + 6 * i + 2);
      const float2 q2 = *reinterpret_cast<const float2*>(d + 6 * i + 4);
      const float du[3] = {q0.x, q0.y, q1.x}, vp[3] = {q1.y, q2.x, q2.y};
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const float wd = wv * du[r];
        a[r * 4 + 0] = fmaf(wd, vp[0], a[r * 4 + 0]);
        a[r * 4 + 1] = fmaf(wd, vp[1], a[r * 4 + 1]);
        a[r * 4 + 2] = fmaf(wd, vp[2], a[r * 4 + 2]);
        a[r * 4 + 3] += wd;
        su[r] += du[r];
      }
    }
    const int hand = g0 + h;
    if (hand < p.n) {
      float* o = p.ws + ((size_t)hand * NCHUNK + blockIdx.y) * WS_STRIDE;
#pragma unroll
      for (int e = 0; e < 12; ++e) o[WS_DA + j * 12 + e] = a[e];
      if (j == 0) { o[WS_DU + 0] = su[0]; o[WS_DU + 1] = su[1]; o[WS_DU + 2] = su[2]; }
    }
  }
  // ---- dpm per (coordinate, row): the row is streamed from L2 (16-byte loads; the model's zero padding and the
  //      zero cotangent of the tail threads cover the rounded-up length), the HG cotangents are broadcast
  {
    const int nv4 = (nv + 3) & ~3;
    for (int task = t; task < 3 * NK; task += VPB) {
      const int c = task / NK, k = task - c * NK;
      const float* __restrict__ dr = m + OFF_DIRS + ((size_t)k * 3 + c) * NVP + v0;
      const float* dv = s_dvp + c * VPB * HG;
      float s[HG];
#pragma unroll
      for (int h = 0; h < HG; ++h) s[h] = 0.f;
      for (int i = 0; i < nv4; i += 4) {
        const float4 d4 = __ldg(reinterpret_cast<const float4*>(dr + i));
        const float dd[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const float4 x0 = *reinterpret_cast<const float4*>(dv + (i + u) * HG);
          const float4 x1 = *reinterpret_cast<const float4*>(dv + (i + u) * HG + 4);
          s[0] = fmaf(dd[u], x0.x, s[0]); s[1] = fmaf(dd[u], x0.y, s[1]);
          s[2] = fmaf(dd[u], x0.z, s[2]); s[3] = fmaf(dd[u], x0.w, s[3]);
          s[4] = fmaf(dd[u], x1.x, s[4]); s[5] = fmaf(dd[u], x1.y, s[5]);
          s[6] = fmaf(dd[u], x1.z, s[6]); s[7] = fmaf(dd[u], x1.w, s[7]);
        }
      }
      float4* o = reinterpret_cast<float4*>(s_dpm3 + (c * NK + k) * HG);
      o[0] = make_float4(s[0], s[1], s[2], s[3]);
      o[1] = make_float4(s[4], s[5], s[6], s[7]);
    }
  }
  __syncthreads();
  for (int task = t; task < NK * HG; task += VPB) {
    const int h = task / NK, k = task - h * NK;
    const int hand = g0 + h;
    if (hand >= p.n) continue;
    const float v = s_dpm3[(0 * NK + k) * HG + h] + s_dpm3[(1 * NK + k) * HG + h] + s_dpm3[(2 * NK + k) * HG + h];
    p.ws[((size_t)hand * NCHUNK + blockIdx.y) * WS_STRIDE + WS_DPM + k] = v;
  }
}

// kPose / kPalm as in mano_forward_body.  With the palm, the kinematic joint 0 is no output: its cotangent reached
// the two palm vertices in the vertex kernel, so it is neither the wrist's dt nor part of the centre term here.
// With POSE_ROTMAT, the rotation cotangent goes through the SO(3) projection's VJP into dposes (n,16,3,3).
template <int kPose, bool kPalm>
__device__ __forceinline__ void mano_backward_chain_body(const ManoGradParams p) {
  __shared__ __align__(16) float s_pm[NK][HG];
  __shared__ __align__(16) float s_A[HG][16][12];
  __shared__ float s_R[HG][16][9];
  __shared__ float s_J[HG][16][3];
  __shared__ float s_G[HG][16][12];
  __shared__ float s_ctr[HG][3];
  __shared__ float s_dG[HG][16][12];     // cotangent of the global transforms [R_g | t_g]
  __shared__ float s_dJ[HG][16][3];      // cotangent of the rest joints
  __shared__ float s_dR[HG][16][9];      // cotangent of the local rotations (chain part)
  __shared__ float s_root[HG][5][15];    // per finger: its level-1 contribution to dG_0 (12) and dJ_0 (3)
  __shared__ float s_dctr[HG][3];

  const int t = threadIdx.x, h = t >> 4, j = t & 15;
  const int hand = blockIdx.x * HG + h;
  const bool valid = hand < p.n;
  rebuild_transforms<true, kPose>(valid, p.model, p.poses, p.betas, hand, h, j, p.center_src, s_pm, s_A, s_R, s_J, s_G,
                                  s_ctr);
  const float* __restrict__ m = p.model;
  // ---- partials of the vertex kernel, summed over the chunks in order
  float dA[12], dpm[9], dpb = 0.f;
#pragma unroll
  for (int e = 0; e < 12; ++e) dA[e] = 0.f;
#pragma unroll
  for (int e = 0; e < 9; ++e) dpm[e] = 0.f;
  if (valid && p.have_partials) {
    for (int ch = 0; ch < NCHUNK; ++ch) {
      const float* w = p.ws + ((size_t)hand * NCHUNK + ch) * WS_STRIDE;
#pragma unroll
      for (int e = 0; e < 12; ++e) dA[e] += w[WS_DA + j * 12 + e];
      if (j >= 1) {
#pragma unroll
        for (int e = 0; e < 9; ++e) dpm[e] += w[WS_DPM + (j - 1) * 9 + e];
      }
      if (j < 10) dpb += w[WS_DPM + 135 + j];
    }
  }
  // ---- centre: d ctr = dcenter - sum(dverts) - sum(djoints)  (every output had the centre subtracted)
  if (j < 3) {
    float d = 0.f;
    if (valid && p.center_src >= 0) {
      if (p.dcenter) d = p.dcenter[(size_t)hand * 3 + j];
      if (p.have_partials)   // sum of du = dverts + fingertip joint cotangents
        for (int ch = 0; ch < NCHUNK; ++ch) d -= p.ws[((size_t)hand * NCHUNK + ch) * WS_STRIDE + WS_DU + j];
      if (p.djoints)
        for (int s = kPalm ? 1 : 0; s < 16; ++s) d -= p.djoints[((size_t)hand * 21 + c_joint_inv[s]) * 3 + j];
    }
    s_dctr[h][j] = d;
  }
  __syncthreads();
  // ---- A_j = [R_g | t_g - R_g J_j]  and the kinematic joint outputs t_g (- ctr)
  {
    const float* G = s_G[h][j];
    float dt[3] = {0.f, 0.f, 0.f};
    if (valid && p.djoints && !(kPalm && j == 0)) {
      const float* d = p.djoints + ((size_t)hand * 21 + c_joint_inv[j]) * 3;
      dt[0] = d[0]; dt[1] = d[1]; dt[2] = d[2];
    }
    if (j == p.center_src) { dt[0] += s_dctr[h][0]; dt[1] += s_dctr[h][1]; dt[2] += s_dctr[h][2]; }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
      for (int c = 0; c < 3; ++c) s_dG[h][j][r * 4 + c] = dA[r * 4 + c] - dA[r * 4 + 3] * s_J[h][j][c];
      s_dG[h][j][r * 4 + 3] = dt[r] + dA[r * 4 + 3];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c)
      s_dJ[h][j][c] = -(G[0 * 4 + c] * dA[0 * 4 + 3] + G[1 * 4 + c] * dA[1 * 4 + 3] + G[2 * 4 + c] * dA[2 * 4 + 3]);
  }
  __syncthreads();
  // ---- chain backward: thread j<5 walks finger j from the tip to the root
  if (j < 5) {
    float dN[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) dN[e] = s_dG[h][3 * j + 3][e];
#pragma unroll
    for (int lev = 2; lev >= 0; --lev) {
      const int idx = 3 * j + 1 + lev, parent = lev ? idx - 1 : 0;
      const float* Gp = s_G[h][parent];
      const float* Rl = s_R[h][idx];
      const float rel[3] = {s_J[h][idx][0] - s_J[h][parent][0], s_J[h][idx][1] - s_J[h][parent][1],
                            s_J[h][idx][2] - s_J[h][parent][2]};
      // N = Gp [Rl | rel] + [0 | t_p]:  dRl = Gp^T dN[:, :3], drel = Gp^T dN[:, 3]
#pragma unroll
      for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
          s_dR[h][idx][i * 3 + c] = Gp[0 * 4 + i] * dN[0 * 4 + c] + Gp[1 * 4 + i] * dN[1 * 4 + c] + Gp[2 * 4 + i] * dN[2 * 4 + c];
      }
      float drel[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) drel[i] = Gp[0 * 4 + i] * dN[0 * 4 + 3] + Gp[1 * 4 + i] * dN[1 * 4 + 3] + Gp[2 * 4 + i] * dN[2 * 4 + 3];
      // dGp[:, :3] = dN[:, :3] Rl^T + dN[:, 3] rel^T,  dGp[:, 3] = dN[:, 3]
      float dP[12];
#pragma unroll
      for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int i = 0; i < 3; ++i)
          dP[r * 4 + i] = dN[r * 4 + 0] * Rl[i * 3 + 0] + dN[r * 4 + 1] * Rl[i * 3 + 1] + dN[r * 4 + 2] * Rl[i * 3 + 2] +
                          dN[r * 4 + 3] * rel[i];
        dP[r * 4 + 3] = dN[r * 4 + 3];
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) s_dJ[h][idx][c] += drel[c];
      if (lev) {
#pragma unroll
        for (int c = 0; c < 3; ++c) s_dJ[h][parent][c] -= drel[c];
#pragma unroll
        for (int e = 0; e < 12; ++e) dN[e] = s_dG[h][parent][e] + dP[e];
      } else {
#pragma unroll
        for (int e = 0; e < 12; ++e) s_root[h][j][e] = dP[e];
#pragma unroll
        for (int c = 0; c < 3; ++c) s_root[h][j][12 + c] = -drel[c];
      }
    }
  }
  __syncthreads();
  // ---- root G_0 = [R_0 | J_0]: the five fingers' contributions in order
  if (j == 0) {
    float dG0[12], dJ0[3];
#pragma unroll
    for (int e = 0; e < 12; ++e) dG0[e] = s_dG[h][0][e];
#pragma unroll
    for (int c = 0; c < 3; ++c) dJ0[c] = s_dJ[h][0][c];
    for (int f = 0; f < 5; ++f) {
#pragma unroll
      for (int e = 0; e < 12; ++e) dG0[e] += s_root[h][f][e];
#pragma unroll
      for (int c = 0; c < 3; ++c) dJ0[c] += s_root[h][f][12 + c];
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
      for (int c = 0; c < 3; ++c) s_dR[h][0][r * 3 + c] = dG0[r * 4 + c];
      s_dJ[h][0][r] = dJ0[r] + dG0[r * 4 + 3];
    }
  }
  __syncthreads();
  if (!valid) return;
  // ---- Rodrigues / SO(3) projection backward (pose map = R - I for joints 1..15)
  if (p.dposes) {
    float g[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) g[e] = s_dR[h][j][e] + dpm[e];
    if constexpr (kPose == POSE_ROTMAT) {
      const size_t off = ((size_t)hand * 16 + j) * 9;
      float dM[9];
      so3_project_vjp(p.poses + off, g, dM);
#pragma unroll
      for (int e = 0; e < 9; ++e) p.dposes[off + e] = dM[e];
    } else {
      const float* ps = p.poses + (size_t)hand * 48 + j * 3;
      float da[3];
      rodrigues_vjp(ps[0] + m[OFF_HM + j * 3 + 0], ps[1] + m[OFF_HM + j * 3 + 1], ps[2] + m[OFF_HM + j * 3 + 2], g, da);
      float* o = p.dposes + (size_t)hand * 48 + j * 3;
      o[0] = da[0]; o[1] = da[1]; o[2] = da[2];
    }
  }
  // ---- betas: the shape rows of the vertices plus J = JT + JS . beta
  if (p.dbetas && j < 10) {
    float d = dpb;
    for (int s = 0; s < 16; ++s)
#pragma unroll
      for (int c = 0; c < 3; ++c) d = fmaf(m[OFF_JS + (s * 3 + c) * 10 + j], s_dJ[h][s][c], d);
    p.dbetas[(size_t)hand * 10 + j] = d;
  }
}

__global__ void __launch_bounds__(VPB) mano_backward_vertex_kernel(const ManoGradParams p) {
  mano_backward_vertex_body<POSE_AXISANG, false>(p);
}
__global__ void __launch_bounds__(VPB) mano_backward_chain_kernel(const ManoGradParams p) {
  mano_backward_chain_body<POSE_AXISANG, false>(p);
}

// the other forms of acr_b200_mano_layer_backward
template <int kPose, bool kPalm>
__global__ void __launch_bounds__(VPB) mano_layer_backward_vertex_kernel(const ManoGradParams p) {
  mano_backward_vertex_body<kPose, kPalm>(p);
}
template <int kPose, bool kPalm>
__global__ void __launch_bounds__(VPB) mano_layer_backward_chain_kernel(const ManoGradParams p) {
  mano_backward_chain_body<kPose, kPalm>(p);
}

// --------------------------------------------------------------------------------------------------- MANO JVP
// Forward-mode derivative of acr_b200_mano_layer_forward: NT tangents of each hand per CTA, no atomics, and every
// tangent runs the same instructions in the same order whatever its slot in a tile, so its result does not depend on
// n_tan or on which tangents share its CTA.
//   phase 1 (thread = (hand, joint)): the primal transforms (rebuild_transforms), then per tangent the rotation
//     tangent dR_j, dJ = JS . dbeta, the chain tangents dG (three levels per finger) and dA_j, all in shared memory;
//   phase 2, full form (thread = vertex): d v_posed = sum_k dirs_k dpm_k, d vert = dT [v_posed; 1] + T d v_posed;
//   phase 2, joints-only form (thread = (hand, tip or palm vertex)): the same for the five tips and the palm only.
constexpr int NT = 4;                 // tangents per CTA (the tangent arrays below take 51.8 KB of shared memory)
constexpr int JCOLS = NT * HG;        // columns (tangent, hand) of the blend-row tangents, [k][t * HG + h]
constexpr int TS_DPM = 0;                             // [NK][JCOLS]         d pm: dR_j (j >= 1) and dbeta
constexpr int TS_DG = TS_DPM + NK * JCOLS;            // [NT][HG][16][12]    dG, then dA in place
constexpr int TS_DJ = TS_DG + NT * HG * 16 * 12;      // [NT][HG][16][3]     d rest joints
constexpr int TS_DR0 = TS_DJ + NT * HG * 16 * 3;      // [NT][HG][9]         dR of the root
constexpr int TS_DCTR = TS_DR0 + NT * HG * 9;         // [NT][HG][3]         d centre
constexpr int TS_PALM = TS_DCTR + NT * HG * 3;        // [NT + 1][HG][2][3]  palm vertices (slot NT: the primal)
constexpr int TS_FLOATS = TS_PALM + (NT + 1) * HG * 6;
constexpr size_t JVP_DYN_SMEM = (size_t)TS_FLOATS * sizeof(float);
static_assert(TS_DG % 4 == 0 && JCOLS % 16 == 0, "16-byte shared loads");

struct ManoJvpParams {
  const float* model;
  int side;
  const float* poses;
  const float* betas;
  int n;
  int center_src;
  int n_tan;
  const float* tposes;   // (n_tan, n, 48) or (n_tan, n, 16, 3, 3), or null (zero)
  const float* tbetas;   // (n_tan, n, 10), or null
  float* verts;
  float* joints;
  float* center;
  float* tverts;         // (n_tan, n, 778, 3)
  float* tjoints;        // (n_tan, n, 21, 3)
  float* tcenter;        // (n_tan, n, 3)
};

// fingertip vertex of slot 0..4 (manolayer.py:244-247)
__device__ __forceinline__ int tip_vertex(int s, int side) {
  return s == 0 ? 745 : s == 1 ? 317 : s == 2 ? (side ? 444 : 445) : s == 3 ? 556 : 673;
}

// a vertex and its tangent from the skinning transform T, its tangent dT, v_posed and d v_posed; explicit FMAs, so
// both JVP forms produce the same bits
__device__ __forceinline__ float vert_row(const float (&T)[12], int r, const float (&vp)[3], float ctr) {
  return fmaf(T[r * 4 + 2], vp[2], fmaf(T[r * 4 + 1], vp[1], fmaf(T[r * 4 + 0], vp[0], T[r * 4 + 3]))) - ctr;
}
__device__ __forceinline__ float tan_row(const float (&T)[12], const float (&dT)[12], int r, const float (&vp)[3],
                                         const float (&dvp)[3], float dctr) {
  float a = dT[r * 4 + 3];
  a = fmaf(dT[r * 4 + 0], vp[0], a); a = fmaf(dT[r * 4 + 1], vp[1], a); a = fmaf(dT[r * 4 + 2], vp[2], a);
  a = fmaf(T[r * 4 + 0], dvp[0], a); a = fmaf(T[r * 4 + 1], dvp[1], a); a = fmaf(T[r * 4 + 2], dvp[2], a);
  return a - dctr;
}

// blend-row order of blend_vertex: the shape rows first
__device__ __forceinline__ int blend_row(int kk) { return (kk < 10) ? 135 + kk : kk - 10; }

// d v_posed of vertex column vc for 2 tangents x HG hands (columns c0 .. c0+15 of s_dpm), from zero
__device__ __forceinline__ void blend_tangents(const float* __restrict__ m, int vc, const float* s_dpm, int c0,
                                               float (&acc)[2 * HG][3]) {
  const float* __restrict__ dirs = m + OFF_DIRS;
  unsigned long long acc2[HG][3];
#pragma unroll
  for (int i = 0; i < HG; ++i) acc2[i][0] = acc2[i][1] = acc2[i][2] = 0ull;   // +0.f pairs
#pragma unroll 5
  for (int kk = 0; kk < NK; ++kk) {
    const int k = blend_row(kk);
    const float d0 = __ldg(dirs + ((size_t)k * 3 + 0) * NVP + vc);
    const float d1 = __ldg(dirs + ((size_t)k * 3 + 1) * NVP + vc);
    const float d2 = __ldg(dirs + ((size_t)k * 3 + 2) * NVP + vc);
    const float4* row = reinterpret_cast<const float4*>(s_dpm + k * JCOLS + c0);
    const unsigned long long D0 = pk2(d0, d0), D1 = pk2(d1, d1), D2 = pk2(d2, d2);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 x = row[q];
      const unsigned long long P0 = pk2(x.x, x.y), P1 = pk2(x.z, x.w);
      ffma2(acc2[2 * q][0], D0, P0); ffma2(acc2[2 * q][1], D1, P0); ffma2(acc2[2 * q][2], D2, P0);
      ffma2(acc2[2 * q + 1][0], D0, P1); ffma2(acc2[2 * q + 1][1], D1, P1); ffma2(acc2[2 * q + 1][2], D2, P1);
    }
  }
#pragma unroll
  for (int i = 0; i < HG; ++i)
#pragma unroll
    for (int c = 0; c < 3; ++c) unpk2(acc2[i][c], acc[2 * i][c], acc[2 * i + 1][c]);
}

// Phase 1 of both JVP forms.  `writer`: this CTA writes the kinematic joints and the centre (tangents of its tile;
// the primal too when it is tangent tile 0).  Ends synchronised, with dA_j in place of dG_j.
template <int kPose, bool kPalm>
__device__ __forceinline__ void jvp_transforms(const ManoJvpParams& p, bool writer, float (*s_pm)[HG],
                                               float (*s_A)[16][12], float (*s_R)[16][9], float (*s_J)[16][3],
                                               float (*s_G)[16][12], float (*s_ctr)[3], float* s_t) {
  const int g0 = blockIdx.x * HG, tile0 = blockIdx.y * NT;
  const int t = threadIdx.x, h = t >> 4, j = t & 15;
  const int hand = g0 + h;
  const bool hvalid = hand < p.n;
  const float* __restrict__ m = p.model;
  rebuild_transforms<true, kPose>(hvalid, m, p.poses, p.betas, hand, h, j, p.center_src, s_pm, s_A, s_R, s_J, s_G,
                                  s_ctr);
  if (writer && hvalid && blockIdx.y == 0) {
    const float* G = s_G[h][j];
    if (p.joints && !(kPalm && j == 0)) {
      float* o = p.joints + ((size_t)hand * 21 + c_joint_inv[j]) * 3;
      o[0] = G[3] - s_ctr[h][0]; o[1] = G[7] - s_ctr[h][1]; o[2] = G[11] - s_ctr[h][2];
    }
    if (j < 3 && p.center) p.center[(size_t)hand * 3 + j] = s_ctr[h][j];
  }
  float* s_dpm = s_t + TS_DPM;
  float* s_dG = s_t + TS_DG;
  float* s_dJ = s_t + TS_DJ;
  float* s_dR0 = s_t + TS_DR0;
  float* s_dctr = s_t + TS_DCTR;
  // ---- per tangent: dR_j, dJ_j = JS_j . dbeta, and the blend-row tangents
  So3ProjectJvp proj;
  if constexpr (kPose == POSE_ROTMAT) {
    if (hvalid && p.tposes) proj.setup(p.poses + ((size_t)hand * 16 + j) * 9);
  }
#pragma unroll 1
  for (int u = 0; u < NT; ++u) {
    const int tt = tile0 + u;
    const bool valid = hvalid && tt < p.n_tan;
    const size_t row = (size_t)tt * p.n + hand;
    const int col = u * HG + h;
    float dR[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (valid && p.tposes) {
      if constexpr (kPose == POSE_ROTMAT) {
        proj.apply(p.tposes + (row * 16 + j) * 9, dR);
      } else {
        const float* ps = p.poses + (size_t)hand * 48 + j * 3;
        rodrigues_jvp(ps[0] + m[OFF_HM + j * 3 + 0], ps[1] + m[OFF_HM + j * 3 + 1], ps[2] + m[OFF_HM + j * 3 + 2],
                      p.tposes + row * 48 + j * 3, dR);
      }
    }
    float dJ[3] = {0.f, 0.f, 0.f};
    if (valid && p.tbetas) {
      const float* db = p.tbetas + row * 10;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float* js = m + OFF_JS + (j * 3 + c) * 10;
        float a = 0.f;
#pragma unroll
        for (int k = 0; k < 10; ++k) a = fmaf(js[k], db[k], a);
        dJ[c] = a;
      }
      if (j < 10) s_dpm[(135 + j) * JCOLS + col] = db[j];
    } else if (j < 10) {
      s_dpm[(135 + j) * JCOLS + col] = 0.f;
    }
#pragma unroll
    for (int e = 0; e < 9; ++e) {
      if (j >= 1) s_dpm[((j - 1) * 9 + e) * JCOLS + col] = dR[e];
      else s_dR0[col * 9 + e] = dR[e];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) s_dJ[(col * 16 + j) * 3 + c] = dJ[c];
    if (j < 3) s_dctr[col * 3 + j] = 0.f;
  }
  __syncthreads();
  // ---- chain tangents: task = (tangent, hand, finger 0..4 or the root 5)
#pragma unroll 1
  for (int task = t; task < NT * HG * 6; task += VPB) {
    const int col = task / 6, f = task - col * 6, hh = col % HG;
    const float* dJ = s_dJ + col * 48;
    float* dG = s_dG + col * 192;
    float dP[12];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      dP[r * 4 + 0] = s_dR0[col * 9 + r * 3 + 0]; dP[r * 4 + 1] = s_dR0[col * 9 + r * 3 + 1];
      dP[r * 4 + 2] = s_dR0[col * 9 + r * 3 + 2]; dP[r * 4 + 3] = dJ[r];
    }
    if (f == 5) {
#pragma unroll
      for (int e = 0; e < 12; ++e) dG[e] = dP[e];
      if (p.center_src == 0) { s_dctr[col * 3 + 0] = dP[3]; s_dctr[col * 3 + 1] = dP[7]; s_dctr[col * 3 + 2] = dP[11]; }
      continue;
    }
    int parent = 0;
#pragma unroll
    for (int lev = 0; lev < 3; ++lev) {
      const int idx = 3 * f + 1 + lev;
      const float* Gp = s_G[hh][parent];
      const float* Rl = s_R[hh][idx];
      float dRl[9];
#pragma unroll
      for (int e = 0; e < 9; ++e) dRl[e] = s_dpm[((idx - 1) * 9 + e) * JCOLS + col];
      const float rel[3] = {s_J[hh][idx][0] - s_J[hh][parent][0], s_J[hh][idx][1] - s_J[hh][parent][1],
                            s_J[hh][idx][2] - s_J[hh][parent][2]};
      const float drel[3] = {dJ[idx * 3 + 0] - dJ[parent * 3 + 0], dJ[idx * 3 + 1] - dJ[parent * 3 + 1],
                             dJ[idx * 3 + 2] - dJ[parent * 3 + 2]};
      // N = Gp [Rl | rel] + [0 | t_p]:  dN = dGp [Rl | rel] + Gp [dRl | drel] + [0 | dt_p]
      float dN[12];
#pragma unroll
      for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
          dN[r * 4 + c] = dP[r * 4 + 0] * Rl[0 * 3 + c] + dP[r * 4 + 1] * Rl[1 * 3 + c] + dP[r * 4 + 2] * Rl[2 * 3 + c] +
                          Gp[r * 4 + 0] * dRl[0 * 3 + c] + Gp[r * 4 + 1] * dRl[1 * 3 + c] + Gp[r * 4 + 2] * dRl[2 * 3 + c];
        dN[r * 4 + 3] = dP[r * 4 + 0] * rel[0] + dP[r * 4 + 1] * rel[1] + dP[r * 4 + 2] * rel[2] +
                        Gp[r * 4 + 0] * drel[0] + Gp[r * 4 + 1] * drel[1] + Gp[r * 4 + 2] * drel[2] + dP[r * 4 + 3];
      }
#pragma unroll
      for (int e = 0; e < 12; ++e) { dP[e] = dN[e]; dG[idx * 12 + e] = dN[e]; }
      if (idx == p.center_src) { s_dctr[col * 3 + 0] = dN[3]; s_dctr[col * 3 + 1] = dN[7]; s_dctr[col * 3 + 2] = dN[11]; }
      parent = idx;
    }
  }
  __syncthreads();
  // ---- kinematic joint and centre tangents, then dA_j = [dR_g | dt_g - dR_g J_j - R_g dJ_j] in place of dG_j
#pragma unroll 1
  for (int u = 0; u < NT; ++u) {
    const int tt = tile0 + u, col = u * HG + h;
    float* dG = s_dG + (col * 16 + j) * 12;
    const float* dJ = s_dJ + (col * 16 + j) * 3;
    const float* dc = s_dctr + col * 3;
    if (writer && hvalid && tt < p.n_tan) {
      const size_t row = (size_t)tt * p.n + hand;
      if (p.tjoints && !(kPalm && j == 0)) {
        float* o = p.tjoints + (row * 21 + c_joint_inv[j]) * 3;
        o[0] = dG[3] - dc[0]; o[1] = dG[7] - dc[1]; o[2] = dG[11] - dc[2];
      }
      if (j < 3 && p.tcenter) p.tcenter[row * 3 + j] = dc[j];
    }
    const float* G = s_G[h][j];
    const float* J = s_J[h][j];
#pragma unroll
    for (int r = 0; r < 3; ++r)
      dG[r * 4 + 3] = dG[r * 4 + 3] - (dG[r * 4 + 0] * J[0] + dG[r * 4 + 1] * J[1] + dG[r * 4 + 2] * J[2]) -
                      (G[r * 4 + 0] * dJ[0] + G[r * 4 + 1] * dJ[1] + G[r * 4 + 2] * dJ[2]);
  }
  __syncthreads();
}

// palm joint (slot NT: the primal, written by tangent tile 0) from the two staged palm vertices of each hand
__device__ __forceinline__ void jvp_write_palm(const ManoJvpParams& p, const float* s_palm) {
  const int g0 = blockIdx.x * HG, tile0 = blockIdx.y * NT;
  for (int task = threadIdx.x; task < (NT + 1) * HG; task += VPB) {
    const int u = task / HG, h = task - u * HG, hand = g0 + h;
    if (hand >= p.n) continue;
    const float* s = s_palm + task * 6;
    float* o;
    if (u == NT) {
      if (blockIdx.y != 0 || !p.joints) continue;
      o = p.joints + (size_t)hand * 21 * 3;
    } else {
      if (tile0 + u >= p.n_tan || !p.tjoints) continue;
      o = p.tjoints + ((size_t)(tile0 + u) * p.n + hand) * 21 * 3;
    }
    o[0] = (s[0] + s[3]) * 0.5f; o[1] = (s[1] + s[4]) * 0.5f; o[2] = (s[2] + s[5]) * 0.5f;
  }
}

// full form: grid (hand groups, tangent tiles, vertex chunks)
template <int kPose, bool kPalm>
__global__ void __launch_bounds__(VPB) mano_layer_jvp_kernel(const ManoJvpParams p) {
  __shared__ __align__(16) float s_pm[NK][HG];
  __shared__ __align__(16) float s_A[HG][16][12];
  __shared__ float s_R[HG][16][9];
  __shared__ float s_J[HG][16][3];
  __shared__ float s_G[HG][16][12];
  __shared__ float s_ctr[HG][3];
  extern __shared__ __align__(16) float s_t[];
  jvp_transforms<kPose, kPalm>(p, blockIdx.z == 0, s_pm, s_A, s_R, s_J, s_G, s_ctr, s_t);
  const float* s_dpm = s_t + TS_DPM;
  const float* s_dA = s_t + TS_DG;
  const float* s_dctr = s_t + TS_DCTR;
  float* s_palm = s_t + TS_PALM;
  const float* __restrict__ m = p.model;
  const int g0 = blockIdx.x * HG, tile0 = blockIdx.y * NT;
  const int v = blockIdx.z * VPB + threadIdx.x;
  const bool vvalid = v < NV;
  const int vc = vvalid ? v : NVP - 1;
  float vp[HG][3];
  blend_vertex(m, vc, s_pm, vp);
  float w[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) w[j] = __ldg(m + OFF_W + j * NVP + vc);
  int tip = -1;
#pragma unroll
  for (int s = 0; s < 5; ++s)
    if (v == tip_vertex(s, p.side)) tip = s;
  const int palm = (kPalm && v == PALM_VA) ? 0 : (kPalm && v == PALM_VB) ? 1 : -1;
  // the primal, from tangent tile 0
  if (blockIdx.y == 0 && (p.verts || p.joints)) {
#pragma unroll
    for (int h = 0; h < HG; ++h) {
      const int hand = g0 + h;
      if (hand >= p.n) continue;                // block-uniform
      float T[12];
      skin_transform(w, s_A[h], T);
      float x[3];
#pragma unroll
      for (int r = 0; r < 3; ++r) x[r] = vert_row(T, r, vp[h], s_ctr[h][r]);
      if (!vvalid) continue;
      if (p.verts) {
        float* o = p.verts + ((size_t)hand * NV + v) * 3;
        o[0] = x[0]; o[1] = x[1]; o[2] = x[2];
      }
      if (tip >= 0 && p.joints) {
        float* o = p.joints + ((size_t)hand * 21 + c_joint_inv[16 + tip]) * 3;
        o[0] = x[0]; o[1] = x[1]; o[2] = x[2];
      }
      if (palm >= 0) {
        float* s = s_palm + (NT * HG + h) * 6 + palm * 3;
        s[0] = x[0]; s[1] = x[1]; s[2] = x[2];
      }
    }
  }
  // the tangents, two per pass
#pragma unroll 1
  for (int pass = 0; pass < NT / 2; ++pass) {
    float dvp[2 * HG][3];
    blend_tangents(m, vc, s_dpm, pass * 2 * HG, dvp);
#pragma unroll
    for (int h = 0; h < HG; ++h) {
      const int hand = g0 + h;
      if (hand >= p.n) continue;                // block-uniform
      float T[12];
      skin_transform(w, s_A[h], T);
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int u = pass * 2 + q, tt = tile0 + u, col = u * HG + h;
        if (tt >= p.n_tan) continue;            // block-uniform
        float dT[12];
        skin_transform(w, reinterpret_cast<const float(*)[12]>(s_dA + col * 192), dT);
        float x[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) x[r] = tan_row(T, dT, r, vp[h], dvp[q * HG + h], s_dctr[col * 3 + r]);
        if (!vvalid) continue;
        const size_t row = (size_t)tt * p.n + hand;
        if (p.tverts) {
          float* o = p.tverts + (row * NV + v) * 3;
          o[0] = x[0]; o[1] = x[1]; o[2] = x[2];
        }
        if (tip >= 0 && p.tjoints) {
          float* o = p.tjoints + (row * 21 + c_joint_inv[16 + tip]) * 3;
          o[0] = x[0]; o[1] = x[1]; o[2] = x[2];
        }
        if (palm >= 0) {
          float* s = s_palm + col * 6 + palm * 3;
          s[0] = x[0]; s[1] = x[1]; s[2] = x[2];
        }
      }
    }
  }
  if constexpr (kPalm) {
    __syncthreads();
    if (blockIdx.z == 0) jvp_write_palm(p, s_palm);
  }
}

// joints-only form: grid (hand groups, tangent tiles); thread (hand, s) takes tip s < 5 or palm vertex s - 5
template <int kPose, bool kPalm>
__global__ void __launch_bounds__(VPB) mano_layer_jvp_joints_kernel(const ManoJvpParams p) {
  __shared__ __align__(16) float s_pm[NK][HG];
  __shared__ __align__(16) float s_A[HG][16][12];
  __shared__ float s_R[HG][16][9];
  __shared__ float s_J[HG][16][3];
  __shared__ float s_G[HG][16][12];
  __shared__ float s_ctr[HG][3];
  extern __shared__ __align__(16) float s_t[];
  jvp_transforms<kPose, kPalm>(p, true, s_pm, s_A, s_R, s_J, s_G, s_ctr, s_t);
  const float* s_dpm = s_t + TS_DPM;
  const float* s_dA = s_t + TS_DG;
  const float* s_dctr = s_t + TS_DCTR;
  float* s_palm = s_t + TS_PALM;
  const float* __restrict__ m = p.model;
  const int g0 = blockIdx.x * HG, tile0 = blockIdx.y * NT;
  const int h = threadIdx.x >> 4, s = threadIdx.x & 15, hand = g0 + h;
  if (s < (kPalm ? 7 : 5) && hand < p.n) {
    const int v = s < 5 ? tip_vertex(s, p.side) : (s == 5 ? PALM_VA : PALM_VB);
    const float* __restrict__ dirs = m + OFF_DIRS;
    // v_posed and its NT tangents in blend_vertex's / blend_tangents' order of rows and operations
    float vp[3] = {m[OFF_VT + 0 * NVP + v], m[OFF_VT + 1 * NVP + v], m[OFF_VT + 2 * NVP + v]};
    float dvp[NT][3];
#pragma unroll
    for (int u = 0; u < NT; ++u) dvp[u][0] = dvp[u][1] = dvp[u][2] = 0.f;
#pragma unroll 5
    for (int kk = 0; kk < NK; ++kk) {
      const int k = blend_row(kk);
      const float d[3] = {__ldg(dirs + ((size_t)k * 3 + 0) * NVP + v), __ldg(dirs + ((size_t)k * 3 + 1) * NVP + v),
                          __ldg(dirs + ((size_t)k * 3 + 2) * NVP + v)};
      const float c = s_pm[k][h];
#pragma unroll
      for (int r = 0; r < 3; ++r) vp[r] = fmaf(d[r], c, vp[r]);
#pragma unroll
      for (int u = 0; u < NT; ++u) {
        const float dc = s_dpm[k * JCOLS + u * HG + h];
#pragma unroll
        for (int r = 0; r < 3; ++r) dvp[u][r] = fmaf(d[r], dc, dvp[u][r]);
      }
    }
    float w[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) w[j] = __ldg(m + OFF_W + j * NVP + v);
    float T[12];
    skin_transform(w, s_A[h], T);
    float x[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) x[r] = vert_row(T, r, vp, s_ctr[h][r]);
    if (s < 5) {
      if (blockIdx.y == 0 && p.joints) {
        float* o = p.joints + ((size_t)hand * 21 + c_joint_inv[16 + s]) * 3;
        o[0] = x[0]; o[1] = x[1]; o[2] = x[2];
      }
    } else {
      float* o = s_palm + (NT * HG + h) * 6 + (s - 5) * 3;
      o[0] = x[0]; o[1] = x[1]; o[2] = x[2];
    }
#pragma unroll
    for (int u = 0; u < NT; ++u) {
      const int tt = tile0 + u, col = u * HG + h;
      if (tt >= p.n_tan) break;
      float dT[12];
      skin_transform(w, reinterpret_cast<const float(*)[12]>(s_dA + col * 192), dT);
#pragma unroll
      for (int r = 0; r < 3; ++r) x[r] = tan_row(T, dT, r, vp, dvp[u], s_dctr[col * 3 + r]);
      if (s < 5) {
        if (p.tjoints) {
          float* o = p.tjoints + (((size_t)tt * p.n + hand) * 21 + c_joint_inv[16 + s]) * 3;
          o[0] = x[0]; o[1] = x[1]; o[2] = x[2];
        }
      } else {
        float* o = s_palm + col * 6 + (s - 5) * 3;
        o[0] = x[0]; o[1] = x[1]; o[2] = x[2];
      }
    }
  }
  if constexpr (kPalm) {
    __syncthreads();
    jvp_write_palm(p, s_palm);
  }
}

}  // namespace acr

using namespace acr;

extern "C" size_t acr_b200_mano_model_floats(void) { return MODEL_FLOATS; }

extern "C" int acr_b200_mano_pack_model(const float* shapedirs, const float* posedirs, const float* v_template,
                                        const float* j_regressor, const float* weights,
                                        const float* hands_mean, int flip_x, float* out) {
  ACR_CHECK_ARG(shapedirs && posedirs && v_template && j_regressor && weights && hands_mean && out,
                "mano_pack_model: null argument");
  for (size_t i = 0; i < MODEL_FLOATS; ++i) out[i] = 0.f;
  auto sd = [&](int v, int c, int k) {
    float s = shapedirs[((size_t)v * 3 + c) * 10 + k];
    return (flip_x && c == 0) ? -s : s;
  };
  for (int v = 0; v < NV; ++v)
    for (int c = 0; c < 3; ++c) {
      for (int k = 0; k < 135; ++k)
        out[OFF_DIRS + ((size_t)k * 3 + c) * NVP + v] = posedirs[((size_t)v * 3 + c) * 135 + k];
      for (int k = 0; k < 10; ++k) out[OFF_DIRS + ((size_t)(135 + k) * 3 + c) * NVP + v] = sd(v, c, k);
      out[OFF_VT + (size_t)c * NVP + v] = v_template[v * 3 + c];
    }
  for (int v = 0; v < NV; ++v)
    for (int j = 0; j < 16; ++j) out[OFF_W + (size_t)j * NVP + v] = weights[v * 16 + j];
  // J = Jreg . (S.beta + T) = (Jreg.S).beta + Jreg.T   -- accumulate in double, store fp32
  for (int j = 0; j < 16; ++j)
    for (int c = 0; c < 3; ++c) {
      double t = 0;
      for (int v = 0; v < NV; ++v) t += (double)j_regressor[(size_t)j * NV + v] * v_template[v * 3 + c];
      out[OFF_JT + j * 3 + c] = (float)t;
      for (int k = 0; k < 10; ++k) {
        double s = 0;
        for (int v = 0; v < NV; ++v) s += (double)j_regressor[(size_t)j * NV + v] * sd(v, c, k);
        out[OFF_JS + (j * 3 + c) * 10 + k] = (float)s;
      }
    }
  for (int i = 0; i < 45; ++i) out[OFF_HM + 3 + i] = hands_mean[i];
  return ACR_B200_OK;
}

static int mano_forward_impl(const float* model_l, const float* model_r, const float* poses,
                             const float* betas, const int32_t* hand_type, int default_side,
                             const int32_t* n_dev, int n_max, int center_idx, const float* cam,
                             const float* offsets, float* verts, float* joints, float* center,
                             float* verts_camed, float* pj2d, float* pj2d_org, const int32_t* counts_src,
                             const acr_b200_gather* g, void* stream) {
  ACR_CHECK_ARG(n_max >= 0, "mano_forward: n_max < 0");
  if (n_max == 0 && !g) return ACR_B200_OK;
  ACR_CHECK_ARG(n_max > 0, "mano_forward_gather: every rank must launch every step (n_max > 0)");
  ACR_CHECK_ARG(poses && betas, "mano_forward: poses/betas are null");
  ACR_CHECK_ARG(default_side == 0 || default_side == 1, "mano_forward: default_side must be 0 or 1");
  ACR_CHECK_ARG(hand_type ? (model_l && model_r) : (default_side ? model_r != nullptr : model_l != nullptr),
                "mano_forward: missing packed model for a requested side");
  ACR_CHECK_ARG(center_idx >= -1 && center_idx < 21, "mano_forward: center_idx out of range");
  ACR_CHECK_ARG(((uintptr_t)verts | (uintptr_t)verts_camed) % 16 == 0, "mano_forward: verts / verts_camed must be 16-byte aligned");
  static const int perm[21] = {0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20};
  int center_src = -1;
  if (center_idx >= 0) {
    center_src = perm[center_idx];
    if (center_src >= 16) {
      set_error("mano_forward: centring on a fingertip joint (center_idx=%d) is not supported", center_idx);
      return ACR_B200_ENOTSUP;
    }
  }
  ManoParams p = {};
  p.model[0] = model_l ? model_l : model_r;
  p.model[1] = model_r ? model_r : model_l;
  p.poses = poses; p.betas = betas; p.hand_type = hand_type; p.default_side = default_side;
  p.n_dev = n_dev; p.n_max = n_max; p.center_src = center_src; p.cam = cam; p.offsets = offsets;
  p.verts = verts; p.joints = joints; p.center = center; p.verts_camed = verts_camed; p.pj2d = pj2d;
  p.pj2d_org = pj2d_org;
  if (g) {
    ACR_CHECK_ARG(g->world >= 1 && g->world <= 8 && g->rank >= 0 && g->rank < g->world, "mano_forward_gather: world / rank");
    ACR_CHECK_ARG(g->rows > 0 && g->rows % 2 == 0 && n_max <= g->rows, "mano_forward_gather: rows per rank must be even and >= n_max");
    ACR_CHECK_ARG(g->slot_bytes % 16 == 0 && g->counts_offset % 16 == 0 && g->flags_offset % 16 == 0 &&
                      g->counts_offset >= (uint64_t)g->world * g->rows * NV * 3 * 4 &&
                      g->slot_bytes >= g->counts_offset + (uint64_t)g->world * 32 && g->flags_offset >= 2 * g->slot_bytes,
                  "mano_forward_gather: slot layout");
    ACR_CHECK_ARG(g->local_state && (uintptr_t)g->local_state % 8 == 0, "mano_forward_gather: local_state");
    p.gather = 1; p.world = g->world; p.rank = g->rank;
    for (int r = 0; r < g->world; ++r) {
      ACR_CHECK_ARG(g->peer_base[r] && g->peer_base[r] % 16 == 0, "mano_forward_gather: peer base %d", r);
      p.peer_base[r] = reinterpret_cast<char*>(g->peer_base[r]);
    }
    p.mc_base = reinterpret_cast<char*>(g->multicast_base);
    p.dst_row = (long long)g->rank * g->rows;
    p.slot_bytes = g->slot_bytes; p.counts_offset = g->counts_offset; p.flags_offset = g->flags_offset;
    p.step_dev = reinterpret_cast<unsigned long long*>(g->local_state);
    p.done_ctr = reinterpret_cast<unsigned int*>(static_cast<char*>(g->local_state) + 8);
    p.counts_src = counts_src;
  }
  dim3 grid(ceil_div(n_max, HG), ceil_div(NV, VPB));
  mano_forward_kernel<<<grid, VPB, 0, (cudaStream_t)stream>>>(p);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

extern "C" int acr_b200_mano_forward(const float* model_l, const float* model_r, const float* poses,
                                     const float* betas, const int32_t* hand_type, int default_side,
                                     const int32_t* n_dev, int n_max, int center_idx, const float* cam,
                                     const float* offsets, float* verts, float* joints, float* center,
                                     float* verts_camed, float* pj2d, float* pj2d_org, void* stream) {
  return mano_forward_impl(model_l, model_r, poses, betas, hand_type, default_side, n_dev, n_max, center_idx, cam,
                           offsets, verts, joints, center, verts_camed, pj2d, pj2d_org, nullptr, nullptr, stream);
}

extern "C" int acr_b200_mano_forward_gather(const float* model_l, const float* model_r, const float* poses,
                                            const float* betas, const int32_t* hand_type, int default_side,
                                            const int32_t* n_dev, int n_max, int center_idx, const float* cam,
                                            const float* offsets, float* verts, float* joints, float* center,
                                            float* verts_camed, float* pj2d, float* pj2d_org,
                                            const int32_t* counts_src, const acr_b200_gather* gather, void* stream) {
  ACR_CHECK_ARG(gather != nullptr, "mano_forward_gather: gather descriptor is null");
  return mano_forward_impl(model_l, model_r, poses, betas, hand_type, default_side, n_dev, n_max, center_idx, cam,
                           offsets, verts, joints, center, verts_camed, pj2d, pj2d_org, counts_src, gather, stream);
}

extern "C" size_t acr_b200_mano_backward_workspace_floats(int n) {
  return n > 0 ? (size_t)n * NCHUNK * WS_STRIDE : 0;
}

extern "C" int acr_b200_mano_backward(const float* model, int side, const float* poses, const float* betas, int n,
                                      int center_idx, const float* dverts, const float* djoints, const float* dcenter,
                                      float* workspace, float* dposes, float* dbetas, void* stream) {
  ACR_CHECK_ARG(n >= 0, "mano_backward: n < 0");
  if (n == 0) return ACR_B200_OK;
  ACR_CHECK_ARG(model && poses && betas, "mano_backward: model / poses / betas are null");
  ACR_CHECK_ARG(side == 0 || side == 1, "mano_backward: side must be 0 (left) or 1 (right)");
  ACR_CHECK_ARG(center_idx >= -1 && center_idx < 21, "mano_backward: center_idx out of range");
  const bool partials = dverts || djoints;
  ACR_CHECK_ARG(!partials || workspace, "mano_backward: workspace is null (acr_b200_mano_backward_workspace_floats)");
  static const int perm[21] = {0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20};
  int center_src = -1;
  if (center_idx >= 0) {
    center_src = perm[center_idx];
    if (center_src >= 16) {
      set_error("mano_backward: centring on a fingertip joint (center_idx=%d) is not supported", center_idx);
      return ACR_B200_ENOTSUP;
    }
  }
  if (!dposes && !dbetas) return ACR_B200_OK;
  ManoGradParams p = {};
  p.model = model; p.side = side; p.poses = poses; p.betas = betas; p.n = n; p.center_src = center_src;
  p.dverts = dverts; p.djoints = djoints; p.dcenter = dcenter; p.ws = workspace; p.have_partials = partials;
  p.dposes = dposes; p.dbetas = dbetas;
  const cudaStream_t s = (cudaStream_t)stream;
  if (partials) {
    static unsigned long long smem_done = 0;
    ACR_CHECK_CUDA(ensure_dynamic_smem(mano_backward_vertex_kernel, (int)GRAD_DYN_SMEM, &smem_done));
    mano_backward_vertex_kernel<<<dim3(ceil_div(n, HG), NCHUNK), VPB, GRAD_DYN_SMEM, s>>>(p);
    ACR_CHECK_LAUNCH();
  }
  mano_backward_chain_kernel<<<ceil_div(n, HG), VPB, 0, s>>>(p);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

// ------------------------------------------------------------------------------------- ManoLayer entry points
// Argument checks shared by acr_b200_mano_layer_forward / _backward -> the centre's source joint (-1 none).
static int layer_args(const char* what, int side, int pose_mode, int center_idx, int root_palm, int* center_src) {
  ACR_CHECK_ARG(side == 0 || side == 1, "%s: side must be 0 (left) or 1 (right)", what);
  ACR_CHECK_ARG(pose_mode == ACR_B200_POSE_AXISANG || pose_mode == ACR_B200_POSE_ROTMAT, "%s: unknown pose_mode %d", what,
                pose_mode);
  ACR_CHECK_ARG(center_idx >= -1 && center_idx < 21, "%s: center_idx out of range", what);
  static const int perm[21] = {0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20};
  *center_src = center_idx >= 0 ? perm[center_idx] : -1;
  if (*center_src >= 16) {
    set_error("%s: centring on a fingertip joint (center_idx=%d) is not supported", what, center_idx);
    return ACR_B200_ENOTSUP;
  }
  if (root_palm && center_idx == 0) {
    set_error("%s: centring on the palm (center_idx=0 with root_palm) is not supported", what);
    return ACR_B200_ENOTSUP;
  }
  return ACR_B200_OK;
}

extern "C" int acr_b200_mano_layer_forward(const float* model, int side, const float* pose, int pose_mode,
                                           const float* betas, int n, int center_idx, int root_palm, float* verts,
                                           float* joints, float* center, void* stream) {
  ACR_CHECK_ARG(n >= 0, "mano_layer_forward: n < 0");
  if (n == 0) return ACR_B200_OK;
  ACR_CHECK_ARG(model && pose && betas, "mano_layer_forward: model / pose / betas are null");
  ACR_CHECK_ARG((uintptr_t)verts % 16 == 0, "mano_layer_forward: verts must be 16-byte aligned");
  int center_src;
  if (const int rc = layer_args("mano_layer_forward", side, pose_mode, center_idx, root_palm, &center_src)) return rc;
  ManoParams p = {};
  p.model[0] = p.model[1] = model;
  p.poses = pose; p.betas = betas; p.default_side = side; p.n_max = n; p.center_src = center_src;
  p.verts = verts; p.joints = joints; p.center = center;
  const dim3 grid(ceil_div(n, HG), ceil_div(NV, VPB));
  const cudaStream_t s = (cudaStream_t)stream;
  if (pose_mode == ACR_B200_POSE_ROTMAT) {
    if (root_palm) mano_layer_forward_kernel<POSE_ROTMAT, true><<<grid, VPB, 0, s>>>(p);
    else mano_layer_forward_kernel<POSE_ROTMAT, false><<<grid, VPB, 0, s>>>(p);
  } else {
    if (root_palm) mano_layer_forward_kernel<POSE_AXISANG, true><<<grid, VPB, 0, s>>>(p);
    else mano_forward_kernel<<<grid, VPB, 0, s>>>(p);
  }
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

template <int kPose, bool kPalm>
static int launch_layer_backward(const ManoGradParams& p, bool partials, cudaStream_t s) {
  if (partials) {
    static unsigned long long smem_done = 0;
    ACR_CHECK_CUDA(ensure_dynamic_smem(mano_layer_backward_vertex_kernel<kPose, kPalm>, (int)GRAD_DYN_SMEM, &smem_done));
    mano_layer_backward_vertex_kernel<kPose, kPalm><<<dim3(ceil_div(p.n, HG), NCHUNK), VPB, GRAD_DYN_SMEM, s>>>(p);
    ACR_CHECK_LAUNCH();
  }
  mano_layer_backward_chain_kernel<kPose, kPalm><<<ceil_div(p.n, HG), VPB, 0, s>>>(p);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

extern "C" int acr_b200_mano_layer_backward(const float* model, int side, const float* pose, int pose_mode,
                                            const float* betas, int n, int center_idx, int root_palm,
                                            const float* dverts, const float* djoints, const float* dcenter,
                                            float* workspace, float* dpose, float* dbetas, void* stream) {
  ACR_CHECK_ARG(n >= 0, "mano_layer_backward: n < 0");
  if (n == 0) return ACR_B200_OK;
  ACR_CHECK_ARG(model && pose && betas, "mano_layer_backward: model / pose / betas are null");
  int center_src;
  if (const int rc = layer_args("mano_layer_backward", side, pose_mode, center_idx, root_palm, &center_src)) return rc;
  const bool partials = dverts || djoints;
  ACR_CHECK_ARG(!partials || workspace, "mano_layer_backward: workspace is null (acr_b200_mano_backward_workspace_floats)");
  if (!dpose && !dbetas) return ACR_B200_OK;
  if (pose_mode == ACR_B200_POSE_AXISANG && !root_palm)
    return acr_b200_mano_backward(model, side, pose, betas, n, center_idx, dverts, djoints, dcenter, workspace, dpose,
                                  dbetas, stream);
  ManoGradParams p = {};
  p.model = model; p.side = side; p.poses = pose; p.betas = betas; p.n = n; p.center_src = center_src;
  p.dverts = dverts; p.djoints = djoints; p.dcenter = dcenter; p.ws = workspace; p.have_partials = partials;
  p.dposes = dpose; p.dbetas = dbetas;
  const cudaStream_t s = (cudaStream_t)stream;
  if (pose_mode == ACR_B200_POSE_ROTMAT)
    return root_palm ? launch_layer_backward<POSE_ROTMAT, true>(p, partials, s)
                     : launch_layer_backward<POSE_ROTMAT, false>(p, partials, s);
  return launch_layer_backward<POSE_AXISANG, true>(p, partials, s);
}

template <int kPose, bool kPalm>
static int launch_layer_jvp(const ManoJvpParams& p, bool full, cudaStream_t s) {
  const dim3 grid(ceil_div(p.n, HG), ceil_div(max(p.n_tan, 1), NT), full ? NCHUNK : 1);
  if (full) {
    static unsigned long long smem_done = 0;
    ACR_CHECK_CUDA(ensure_dynamic_smem(mano_layer_jvp_kernel<kPose, kPalm>, (int)JVP_DYN_SMEM, &smem_done));
    mano_layer_jvp_kernel<kPose, kPalm><<<grid, VPB, JVP_DYN_SMEM, s>>>(p);
  } else {
    static unsigned long long smem_done = 0;
    ACR_CHECK_CUDA(ensure_dynamic_smem(mano_layer_jvp_joints_kernel<kPose, kPalm>, (int)JVP_DYN_SMEM, &smem_done));
    mano_layer_jvp_joints_kernel<kPose, kPalm><<<grid, VPB, JVP_DYN_SMEM, s>>>(p);
  }
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

extern "C" int acr_b200_mano_layer_jvp(const float* model, int side, const float* pose, int pose_mode,
                                       const float* betas, int n, int center_idx, int root_palm, int n_tan,
                                       const float* tpose, const float* tbetas, float* verts, float* joints,
                                       float* center, float* tverts, float* tjoints, float* tcenter, void* stream) {
  ACR_CHECK_ARG(n >= 0, "mano_layer_jvp: n < 0");
  ACR_CHECK_ARG(n_tan >= 0, "mano_layer_jvp: n_tan < 0");
  if (n == 0) return ACR_B200_OK;
  ACR_CHECK_ARG(model && pose && betas, "mano_layer_jvp: model / pose / betas are null");
  ACR_CHECK_ARG(n_tan <= 65535 * NT, "mano_layer_jvp: n_tan > %d", 65535 * NT);
  int center_src;
  if (const int rc = layer_args("mano_layer_jvp", side, pose_mode, center_idx, root_palm, &center_src)) return rc;
  const bool tangents = n_tan > 0 && (tverts || tjoints || tcenter);
  if (!tangents && !verts && !joints && !center) return ACR_B200_OK;
  ManoJvpParams p = {};
  p.model = model; p.side = side; p.poses = pose; p.betas = betas; p.n = n; p.center_src = center_src;
  p.n_tan = tangents ? n_tan : 0; p.tposes = tpose; p.tbetas = tbetas;
  p.verts = verts; p.joints = joints; p.center = center; p.tverts = tverts; p.tjoints = tjoints; p.tcenter = tcenter;
  // without vertices (primal or tangent) one CTA per hand group and tangent tile: the joints-only form
  const bool full = verts || tverts;
  const cudaStream_t s = (cudaStream_t)stream;
  if (pose_mode == ACR_B200_POSE_ROTMAT)
    return root_palm ? launch_layer_jvp<POSE_ROTMAT, true>(p, full, s) : launch_layer_jvp<POSE_ROTMAT, false>(p, full, s);
  return root_palm ? launch_layer_jvp<POSE_AXISANG, true>(p, full, s) : launch_layer_jvp<POSE_AXISANG, false>(p, full, s);
}

extern "C" int acr_b200_gather_wait(const acr_b200_gather* g, void* stream) {
  ACR_CHECK_ARG(g && g->world >= 1 && g->world <= 8 && g->local_state && g->peer_base[g->rank], "gather_wait: bad descriptor");
  gather_wait_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const unsigned long long*>(reinterpret_cast<const char*>(g->peer_base[g->rank]) + g->flags_offset),
      reinterpret_cast<const unsigned long long*>(g->local_state), g->world);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

extern "C" int acr_b200_cam_trans(const float* j3d, const float* pj2d, const int32_t* n_dev, int n_max,
                                  float focal_length, float img_size, float* cam_trans, void* stream) {
  ACR_CHECK_ARG(n_max >= 0 && (n_max == 0 || (j3d && pj2d && cam_trans)), "cam_trans: bad arguments");
  if (n_max == 0) return ACR_B200_OK;
  cam_trans_kernel<<<ceil_div(n_max, 128), 128, 0, (cudaStream_t)stream>>>(j3d, pj2d, n_dev, n_max, focal_length, img_size, cam_trans);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

extern "C" int acr_b200_rot6d_to_aa(const float* rot6d, int n_rot, float* aa, void* stream) {
  ACR_CHECK_ARG(n_rot >= 0 && (n_rot == 0 || (rot6d && aa)), "rot6d_to_aa: bad arguments");
  if (n_rot == 0) return ACR_B200_OK;
  rot6d_to_aa_kernel<<<ceil_div(n_rot, 128), 128, 0, (cudaStream_t)stream>>>(rot6d, n_rot, aa);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}

extern "C" int acr_b200_rodrigues(const float* aa, int n_rot, float* rotmat, void* stream) {
  ACR_CHECK_ARG(n_rot >= 0 && (n_rot == 0 || (aa && rotmat)), "rodrigues: bad arguments");
  if (n_rot == 0) return ACR_B200_OK;
  rodrigues_kernel<<<ceil_div(n_rot, 128), 128, 0, (cudaStream_t)stream>>>(aa, n_rot, rotmat);
  ACR_CHECK_LAUNCH();
  return ACR_B200_OK;
}
