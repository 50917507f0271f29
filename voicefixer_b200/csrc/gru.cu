// Bidirectional GRU layer recurrence (hidden 256), torch.nn.GRU semantics:
//   r = sigmoid(gi_r + W_hr h + b_hr); z = sigmoid(gi_z + W_hz h + b_hz)
//   n = tanh(gi_n + r * (W_hn h + b_hn)); h' = (1 - z) * n + z * h
// Reference: BN_GRU voicefixer/restorer/model.py:22-62 (nn.GRU(512, 256, num_layers=2,
// bidirectional=True, batch_first=True)); state is zero at the start of every segment.
// The input projections gi = x W_ih^T + b_ih are one batched GEMM (conv_gemm); this kernel is the
// sequential part and is latency-bound (T = 1001 .. 3001 dependent steps).
//
// Design (sm_90a): one thread-block CLUSTER of 8 CTAs per (direction, group of G sequences).
//   * W_hh (768 x 256 fp32 = 786 KB) never fits one SM: CTA c owns hidden units [32c, 32c+32), i.e.
//     96 gate rows, and keeps its 96 x 256 slice in REGISTERS (96 per thread) for all T steps, so a
//     step reads no weights from shared memory, L2 or HBM.
//   * every CTA holds a replica of h (double-buffered, G x 256); after computing its 32 x G new
//     values a CTA pushes them into all 8 replicas with st.async (distributed shared memory stores
//     that complete_tx on the DESTINATION CTA's mbarrier); each CTA starts its next step when its
//     own mbarrier has received all 256 x G values.  No cluster barrier and no memory fence per
//     step.
//   * fp32 FMA throughout (the recurrence is precision-sensitive); gi for step t+1 is prefetched
//     into registers during step t.
#include <cooperative_groups.h>
#include <stdlib.h>
#include "vfx_common.cuh"

namespace cg = cooperative_groups;

namespace vfx {

namespace {

constexpr int H = 256, G3 = 768;
constexpr int CL = 8;            // CTAs per cluster
constexpr int UPC = H / CL;      // hidden units per CTA = 32
constexpr int RPC = 3 * UPC;     // gate rows per CTA = 96
// K split: one H/KQ-wide slice per warp, KQ warps per CTA (lane = hidden unit of this CTA, warp = K slice).
// KQ = 8 (default): 256 threads x 96 weights; KQ = 16 (VFX_GRU_KQ=16): 512 threads x 48 weights -- same total work, twice
// the warps.  An ncu capture of KQ = 8 shows 25 % issue-active and 24 % of samples in the mbarrier wait of the exchange;
// doubling the warps did not shorten the step (see gru_layer below), so the default stays at 8.

template <int G, int KQ>
__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(32 * KQ, 1)
gru_cluster_kernel(const float* __restrict__ gi, const float* __restrict__ whh_t,
                   const float* __restrict__ bhh, int B, int T, const int* __restrict__ lens, float* __restrict__ out) {
  constexpr int KW = H / KQ, NT = 32 * KQ;
  extern __shared__ __align__(16) uint8_t gru_smem[];
  float (*h_s)[G][H] = reinterpret_cast<float (*)[G][H]>(gru_smem);                       // [2][G][H]
  float (*part)[KQ][G][RPC] = reinterpret_cast<float (*)[KQ][G][RPC]>(gru_smem + sizeof(float) * 2 * G * H);
  uint64_t* hbar = reinterpret_cast<uint64_t*>(gru_smem + sizeof(float) * (2 * G * H + 2 * KQ * G * RPC));
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int cl = blockIdx.x / CL;
  const int dir = cl & 1;
  const int b0 = (cl >> 1) * G;
  const int tid = threadIdx.x;
  const int q = tid >> 5, u = tid & 31;                   // K slice, hidden unit (of this CTA)

  // this thread's 96 weights: the r/z/n rows of unit (rank*32 + u), columns [q*32, q*32+32)
  // (whh_t is [dir][k][768]: coalesced over u).  All lanes of a warp share the K slice, so the h
  // loads below are pure shared-memory broadcasts, each feeding 12 FMAs.
  float w[3][KW];
  {
    const float* W = whh_t + (long long)dir * H * G3 + (long long)(q * KW) * G3 + rank * UPC + u;
#pragma unroll
    for (int g3 = 0; g3 < 3; ++g3)
#pragma unroll
      for (int i = 0; i < KW; ++i) w[g3][i] = W[(long long)i * G3 + g3 * H];
  }
  // finaliser role: thread (fg, fu) produces h'[fg][rank*32 + fu]
  const bool fin = tid < UPC * G;
  const int fu = tid % UPC, fg = tid / UPC;
  const bool fvalid = fin && (b0 + fg) < B;
  // ragged batch: this item's own length; its backward direction starts at Tb - 1 and steps >= Tb store nothing
  const int Tb = fvalid && lens ? lens[b0 + fg] : T;
  const int hu = rank * UPC + fu;
  float b_r = 0.f, b_z = 0.f, b_n = 0.f;
  if (fin) {
    const float* bb = bhh + dir * G3 + hu;
    b_r = bb[0]; b_z = bb[H]; b_n = bb[2 * H];
  }
  // shared::cluster addresses of every replica's h buffer and mbarriers
  uint32_t rem_h[CL], rem_bar[CL];
  {
    const uint32_t lh = (uint32_t)__cvta_generic_to_shared(&h_s[0][0][0]);
    const uint32_t lb = (uint32_t)__cvta_generic_to_shared(&hbar[0]);
#pragma unroll
    for (int c = 0; c < CL; ++c) {
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rem_h[c]) : "r"(lh), "r"(c));
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rem_bar[c]) : "r"(lb), "r"(c));
    }
  }
  for (int i = tid; i < 2 * G * H; i += NT) (&h_s[0][0][0])[i] = 0.f;
  if (tid == 0) {
    const uint32_t lb = (uint32_t)__cvta_generic_to_shared(&hbar[0]);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(lb));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(lb + 8));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  cluster.sync();

  // input projections are prefetched two steps ahead (register ring): an HBM round trip is longer
  // than one step
  const long long gstride = 2LL * G3;                     // floats per (b, t)
  const float* gbase = gi + ((long long)(b0 + fg) * T) * gstride + dir * G3 + hu;
  float pr[2] = {0.f, 0.f}, pz[2] = {0.f, 0.f}, pn[2] = {0.f, 0.f};
#pragma unroll
  for (int s = 0; s < 2; ++s)
    if (fvalid && s < Tb) {
      const int ts = dir == 0 ? s : Tb - 1 - s;
      const float* p = gbase + (long long)ts * gstride;
      pr[s] = p[0]; pz[s] = p[H]; pn[s] = p[2 * H];
    }

  for (int step = 0; step < T; ++step) {
    const int t = dir == 0 ? step : Tb - 1 - step;      // < 0 (backward) or >= Tb (forward) past this item's end
    const int cur = step & 1, nxt = cur ^ 1;
    const bool last = step + 1 == T;
    if (tid == 0 && !last) {      // arm the mbarrier of the buffer this step's exchange fills
      const uint32_t lb = (uint32_t)__cvta_generic_to_shared(&hbar[nxt]);
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(lb), "r"(G * H * 4) : "memory");
    }
    const float gir = pr[0], giz = pz[0], gin = pn[0];
    pr[0] = pr[1]; pz[0] = pz[1]; pn[0] = pn[1];
    if (fvalid && step + 2 < Tb) {
      const int tn = dir == 0 ? t + 2 : t - 2;
      const float* p = gbase + (long long)tn * gstride;
      pr[1] = p[0]; pz[1] = p[H]; pn[1] = p[2 * H];
    }
    // ---- phase A: partial dot products over this thread's K quarter, all G sequences
    float acc[3][G];
#pragma unroll
    for (int g3 = 0; g3 < 3; ++g3)
#pragma unroll
      for (int g = 0; g < G; ++g) acc[g3][g] = 0.f;
#pragma unroll
    for (int i = 0; i < KW; i += 4) {
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const float4 hv = *reinterpret_cast<const float4*>(&h_s[cur][g][q * KW + i]);
#pragma unroll
        for (int g3 = 0; g3 < 3; ++g3) {
          acc[g3][g] = fmaf(w[g3][i], hv.x, acc[g3][g]);
          acc[g3][g] = fmaf(w[g3][i + 1], hv.y, acc[g3][g]);
          acc[g3][g] = fmaf(w[g3][i + 2], hv.z, acc[g3][g]);
          acc[g3][g] = fmaf(w[g3][i + 3], hv.w, acc[g3][g]);
        }
      }
    }
#pragma unroll
    for (int g3 = 0; g3 < 3; ++g3)
#pragma unroll
      for (int g = 0; g < G; ++g) part[cur][q][g][g3 * UPC + u] = acc[g3][g];
    __syncthreads();
    // ---- phase B: gates for 32 units x G sequences, push h' into all 8 replicas
    if (fin) {
      float gr = b_r, gz = b_z, gn = b_n;
#pragma unroll
      for (int k = 0; k < KQ; ++k) {
        gr += part[cur][k][fg][fu]; gz += part[cur][k][fg][UPC + fu]; gn += part[cur][k][fg][2 * UPC + fu];
      }
      const float rg = 1.f / (1.f + expf(-(gir + gr)));
      const float zg = 1.f / (1.f + expf(-(giz + gz)));
      const float ng = tanhf(gin + rg * gn);
      const float hn = (1.f - zg) * ng + zg * h_s[cur][fg][hu];
      if (!last) {
        const uint32_t off = (uint32_t)(((nxt * G + fg) * H + hu) * 4);
#pragma unroll
        for (int c = 0; c < CL; ++c)
          asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];"
                       ::"r"(rem_h[c] + off), "r"(__float_as_uint(hn)), "r"(rem_bar[c] + 8u * nxt) : "memory");
      }
      if (fvalid && step < Tb) out[((long long)(b0 + fg) * T + t) * (2 * H) + dir * H + hu] = hn;
    }
    if (!last) {                  // wait until all 8 CTAs' contributions to h[nxt] have landed here
      const uint32_t lb = (uint32_t)__cvta_generic_to_shared(&hbar[nxt]);
      const uint32_t parity = (uint32_t)((step >> 1) & 1);
      asm volatile(
          "{\n\t.reg .pred p;\n\t"
          "GRU_WAIT:\n\t"
          "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
          "@p bra GRU_DONE;\n\t"
          "bra GRU_WAIT;\n\t"
          "GRU_DONE:\n\t}" ::"r"(lb), "r"(parity) : "memory");
    }
  }
  cluster.sync();   // no CTA may exit while a peer could still address its shared memory
}

template <int G, int KQ>
int launch(const float* gi, const float* whh_t, const float* bhh, int B, int T, const int* lens, float* out,
           cudaStream_t st) {
  constexpr int NT = 32 * KQ;
  const int groups = (B + G - 1) / G;
  const size_t smem = sizeof(float) * (2 * G * H + 2 * KQ * G * RPC) + 16;
  static bool attr_set[64] = {false};           // per device: the attribute belongs to the device's copy of the function
  int dev = 0;
  VFX_CUDA_CHECK(cudaGetDevice(&dev));
  if (dev >= 64 || !attr_set[dev]) {
    VFX_CUDA_CHECK(cudaFuncSetAttribute(gru_cluster_kernel<G, KQ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (dev < 64) attr_set[dev] = true;
  }
  gru_cluster_kernel<G, KQ><<<2 * groups * CL, NT, smem, st>>>(gi, whh_t, bhh, B, T, lens, out);
  VFX_LAUNCH_CHECK();
  return VFX_OK;
}

}  // namespace

int gru_layer(const float* gi, const float* whh_t, const float* bhh, int B, int T, const int* lens, float* out,
              cudaStream_t st) {
  VFX_REQUIRE(B > 0 && T > 0, "gru_layer: empty problem");
  // one wave: at most 16 clusters of 8 CTAs (128 of the 132 SMs, two clusters per GPC)
  static const int kq = getenv("VFX_GRU_KQ") ? atoi(getenv("VFX_GRU_KQ")) : 8;
  if (kq == 8) {
    if (2 * ((B + 1) / 2) <= 16) return launch<2, 8>(gi, whh_t, bhh, B, T, lens, out, st);
    if (2 * ((B + 3) / 4) <= 16) return launch<4, 8>(gi, whh_t, bhh, B, T, lens, out, st);
    return launch<8, 8>(gi, whh_t, bhh, B, T, lens, out, st);
  }
  if (2 * ((B + 1) / 2) <= 16) return launch<2, 16>(gi, whh_t, bhh, B, T, lens, out, st);
  if (2 * ((B + 3) / 4) <= 16) return launch<4, 16>(gi, whh_t, bhh, B, T, lens, out, st);
  return launch<8, 16>(gi, whh_t, bhh, B, T, lens, out, st);
}

}  // namespace vfx
