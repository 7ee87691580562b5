// Non-causal multi-head attention forward for sm_90a (head_dim 128), flash-style, on wgmma.
//
//   out[b, i, h*128:(h+1)*128] = softmax_j( q[b,i,h,:] . k[b,j,h,:] * scale ) @ v[b,j,h,:]
//
// One CTA per (128-query tile, head, batch); 384 threads = 3 warpgroups (registers re-partitioned with setmaxnreg):
//   warpgroup 0     TMA producer (one lane of warp 0): Q tile once, then K_j / V_j tiles (128 keys) through 2-deep rings
//   warpgroups 1,2  one 64-query half of the tile each, everything in registers:
//                   S_j = Q K_j^T (wgmma, both operands from shared memory), online softmax (fp32: running max, exp2, running sum),
//                   O += P_j V_j (wgmma, bf16 P_j straight from the S accumulator registers as the A operand, V_j as MN-major B)
// The two warpgroups run independently, so the softmax of one overlaps the MMAs of the other on the tensor cores.
// With a second key/value source (text + image cross-attention) the same CTA walks the second source after the first and adds
// its separately normalised, bf16-rounded result to the first one's.
//
// Shared memory: Q 32K | K 2x32K | V 2x32K | barriers.
//
// Replaces F.scaled_dot_product_attention at chronoedit_diffusers/transformer_chronoedit.py:91-99 of the reference
// (self-attention, text cross-attention and image cross-attention; the latter two are summed, :103-104).
#include "attention.cuh"
#include "wgmma.cuh"

namespace ce {

namespace {

constexpr int HD = 128;
constexpr int BQ = 128;
constexpr int BKV = 128;
constexpr int ATTN_THREADS = 384;
constexpr uint32_t TILE_BYTES = 128 * 128 * 2;  // 32 KB: two 16 KB [128 x 64] swizzled blocks
constexpr uint32_t HALF_BYTES = TILE_BYTES / 2;

struct SmemLayout {
  static constexpr uint32_t q = 0;
  static constexpr uint32_t k = q + TILE_BYTES;
  static constexpr uint32_t v = k + 2 * TILE_BYTES;
  static constexpr uint32_t bars = v + 2 * TILE_BYTES;
  static constexpr uint32_t total = bars + 256;
};

// barrier indices
enum { Q_FULL = 0, K_FULL = 1, K_EMPTY = 3, V_FULL = 5, V_EMPTY = 7, NUM_BARS = 9 };

__global__ void __launch_bounds__(ATTN_THREADS, 1)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tma_q, const __grid_constant__ CUtensorMap tma_k,
                     const __grid_constant__ CUtensorMap tma_v, const __grid_constant__ CUtensorMap tma_k2,
                     const __grid_constant__ CUtensorMap tma_v2, AttnArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SmemLayout::bars);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * BQ;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  // key tiles of source 0 (k / v, Lk keys), then of source 1 (k2 / v2, Lk2 keys; none for a single source), through one ring
  const int T0 = (a.Lk + BKV - 1) / BKV;
  const int T1 = (a.Lk2 + BKV - 1) / BKV;

  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();  // the swizzled tiles need 1024-byte alignment
    for (int i = 0; i < NUM_BARS; ++i) mbar_init(&bars[i], (i >= K_EMPTY && i < K_EMPTY + 2) || (i >= V_EMPTY && i < V_EMPTY + 2) ? 2 : 1);
    fence_mbar_init();
    tma_prefetch_desc(&tma_q);
    tma_prefetch_desc(&tma_k);
    tma_prefetch_desc(&tma_v);
    tma_prefetch_desc(&tma_k2);
    tma_prefetch_desc(&tma_v2);
  }
  __syncthreads();

  if (warp < 4) {
    // ---------------------------------------------------------------- TMA producer
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one_sync()) {
      mbar_arrive_expect_tx(&bars[Q_FULL], TILE_BYTES);
      tma_load_3d(smem + SmemLayout::q, &tma_q, &bars[Q_FULL], h * HD, q0, b);
      tma_load_3d(smem + SmemLayout::q + HALF_BYTES, &tma_q, &bars[Q_FULL], h * HD + 64, q0, b);
      for (int t = 0; t < T0 + T1; ++t) {
        const int s = t & 1;
        const uint32_t free_parity = ((t >> 1) & 1) ^ 1;
        const CUtensorMap* mk = t < T0 ? &tma_k : &tma_k2;
        const CUtensorMap* mv = t < T0 ? &tma_v : &tma_v2;
        const int row0 = (t < T0 ? t : t - T0) * BKV;
        uint8_t* ks = smem + SmemLayout::k + s * TILE_BYTES;
        uint8_t* vs = smem + SmemLayout::v + s * TILE_BYTES;
        mbar_wait(&bars[K_EMPTY + s], free_parity);
        mbar_arrive_expect_tx(&bars[K_FULL + s], TILE_BYTES);
        tma_load_3d(ks, mk, &bars[K_FULL + s], h * HD, row0, b);
        tma_load_3d(ks + HALF_BYTES, mk, &bars[K_FULL + s], h * HD + 64, row0, b);
        mbar_wait(&bars[V_EMPTY + s], free_parity);
        mbar_arrive_expect_tx(&bars[V_FULL + s], TILE_BYTES);
        tma_load_3d(vs, mv, &bars[V_FULL + s], h * HD, row0, b);
        tma_load_3d(vs + HALF_BYTES, mv, &bars[V_FULL + s], h * HD + 64, row0, b);
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumers: 64 query rows per warpgroup
  setmaxnreg_inc<232>();
  const int wg = (warp >> 2) - 1;
  const bool signaller = (threadIdx.x & 127) == 0;
  const int quad = lane & 3;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // the thread's rows of the query tile: r0 and r0 + 8
  const float sl2 = a.scale * 1.4426950408889634f;
  const uint32_t q_smem = smem_u32(smem + SmemLayout::q) + wg * 64 * 128;
  const bool timed = a.timing != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && threadIdx.x == 128;
  long long tacc[3] = {0, 0, 0};   // cycles in S = Q K^T (incl. the wait for K), softmax, P V (incl. the wait for V)
  long long tc0 = timed ? clock64() : 0;
#define CE_TICK(slot)               \
  if (timed) {                      \
    const long long _t = clock64(); \
    tacc[slot] += _t - tc0;         \
    tc0 = _t;                       \
  }

  mbar_wait(&bars[Q_FULL], 0);
  int t = 0;   // position in the ring, over both sources
  for (int src = 0; src < (T1 > 0 ? 2 : 1); ++src) {
    const int my_tiles = src ? T1 : T0;
    const int my_len = src ? a.Lk2 : a.Lk;
    float o[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // per row; l is this lane's share of the row sum

    for (int j = 0; j < my_tiles; ++j, ++t) {
      const int s = t & 1;
      const uint32_t parity = (t >> 1) & 1;
      const int valid = my_len - j * BKV;  // >= 1; >= 128 means no masking
      // ---- S = Q K^T: 8 K16 steps over head_dim (two 64-wide swizzled blocks)
      float sc[64];
      mbar_wait(&bars[K_FULL + s], parity);
      {
        const uint32_t k_smem = smem_u32(smem + SmemLayout::k) + s * TILE_BYTES;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
          const uint32_t off = (kk >> 2) * HALF_BYTES + (kk & 3) * 32;
          wgmma_ss<128, 0>(sc, wgmma_desc_kmajor_sw128(q_smem + off), wgmma_desc_kmajor_sw128(k_smem + off), kk != 0);
        }
        wgmma_commit();
        wgmma_wait<0>();
        if (signaller) mbar_arrive(&bars[K_EMPTY + s]);
      }
      CE_TICK(0)
      // ---- online softmax on the accumulator registers: sc[4 * c + e + 2 * hh] is row r0 + 8 * hh, key 8 * c + 2 * quad + e
      if (valid < BKV) {  // last key tile only (warp-uniform): masked scores -> -inf -> p = 0
#pragma unroll
        for (int i = 0; i < 64; ++i)
          if (8 * (i >> 2) + 2 * quad + (i & 1) >= valid) sc[i] = -INFINITY;
      }
      uint32_t p[32];   // bf16 pairs: p[2 * c + hh] = keys 8 * c + 2 * quad + {0, 1} of row r0 + 8 * hh
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float mx = -INFINITY;
#pragma unroll
        for (int c = 0; c < 16; ++c) mx = fmaxf(mx, fmaxf(sc[4 * c + 2 * hh], sc[4 * c + 2 * hh + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m[hh], mx * sl2);   // finite: every tile has at least one valid key
        const float alpha = fast_exp2(m[hh] - m_new); // 0 on the first tile (m = -inf)
        m[hh] = m_new;
        float sum = 0.f;
#pragma unroll
        for (int c = 0; c < 16; ++c) {
          const float p0 = fast_exp2(fmaf(sc[4 * c + 2 * hh], sl2, -m_new));
          const float p1 = fast_exp2(fmaf(sc[4 * c + 2 * hh + 1], sl2, -m_new));
          sum += p0 + p1;
          p[2 * c + hh] = pack_bf16x2(p0, p1);
        }
        l[hh] = l[hh] * alpha + sum;
#pragma unroll
        for (int c = 0; c < 16; ++c) {
          o[4 * c + 2 * hh] *= alpha;
          o[4 * c + 2 * hh + 1] *= alpha;
        }
      }
      CE_TICK(1)
      // ---- O += P V: 8 K16 steps over the keys; the A fragment of step kk is {rows r0, r0+8} x {keys 16kk + 2quad, + 8}
      mbar_wait(&bars[V_FULL + s], parity);
      {
        const uint32_t v_smem = smem_u32(smem + SmemLayout::v) + s * TILE_BYTES;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
          const uint32_t frag[4] = {p[4 * kk], p[4 * kk + 1], p[4 * kk + 2], p[4 * kk + 3]};
          wgmma_rs<128, 1>(o, frag, wgmma_desc_mnmajor_sw128(v_smem + kk * 2048, HALF_BYTES), 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
        if (signaller) mbar_arrive(&bars[V_EMPTY + s]);
      }
      CE_TICK(2)
    }

    // ---- normalise and store this source's result
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float lr = l[hh];
      lr += __shfl_xor_sync(0xffffffffu, lr, 1);
      lr += __shfl_xor_sync(0xffffffffu, lr, 2);
      const float inv = 1.0f / lr;
      const int row = q0 + r0 + 8 * hh;
      if (row >= a.Lq) continue;
      bf16* orow = a.out + ((size_t)b * a.Lq + row) * a.ldo + h * HD;
      if (a.peer_rows > 0)   // sequence parallel: the token's owner gets the row (peer store over NVLink)
        orow = a.out_peer[row / a.peer_rows] + ((size_t)b * a.peer_rows + row % a.peer_rows) * a.ldo + a.out_col0 + h * HD;
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        float y0 = o[4 * c + 2 * hh] * inv, y1 = o[4 * c + 2 * hh + 1] * inv;
        uint32_t* dst = reinterpret_cast<uint32_t*>(orow + 8 * c + 2 * quad);
        if (a.accumulate || src == 1) {   // each SDPA result is a bf16 tensor in the reference before the add
          const float2 prev = unpack_bf16x2(*dst);
          y0 = bf16_round(y0) + prev.x;
          y1 = bf16_round(y1) + prev.y;
        }
        *dst = pack_bf16x2(y0, y1);
      }
    }
  }
  if (timed) {
    for (int i = 0; i < 3; ++i) a.timing[i] = tacc[i];
    a.timing[3] = T0 + T1;
  }
#undef CE_TICK
}


int make_qkv_tmap(CUtensorMap* m, const bf16* base, int B, int L, int H, int ld) {
  uint64_t dims[3] = {(uint64_t)H * HD, (uint64_t)L, (uint64_t)B};
  uint64_t strides[2] = {(uint64_t)ld * 2, (uint64_t)L * ld * 2};
  uint32_t box[3] = {64, 128, 1};
  return make_tmap_bf16(m, base, 3, dims, strides, box);
}

}  // namespace

int launch_attention(const AttnArgs& a, cudaStream_t stream) {
  CE_REQUIRE(a.B > 0 && a.H > 0 && a.Lq > 0 && a.Lk > 0, "attention: empty problem");
  CE_REQUIRE(a.peer_rows == 0 || (a.Lk2 == 0 && !a.accumulate && (a.Lq + a.peer_rows - 1) / a.peer_rows <= 8),
             "attention: the sequence-parallel output scatter serves the self-attention, with at most 8 peers");
  CE_REQUIRE(a.head_dim == HD, "attention: only head_dim 128 is built");
  CE_REQUIRE(a.ldq % 8 == 0 && a.ldk % 8 == 0 && a.ldv % 8 == 0 && a.ldo % 8 == 0, "attention: leading dims % 8");
  CE_REQUIRE(a.q && a.k && a.v && a.out, "attention: null pointer");
  CUtensorMap tq, tk, tv, tk2, tv2;
  int rc;
  if ((rc = make_qkv_tmap(&tq, a.q, a.B, a.Lq, a.H, a.ldq))) return rc;
  if ((rc = make_qkv_tmap(&tk, a.k, a.B, a.Lk, a.H, a.ldk))) return rc;
  if ((rc = make_qkv_tmap(&tv, a.v, a.B, a.Lk, a.H, a.ldv))) return rc;
  if (a.Lk2 > 0) {
    CE_REQUIRE(a.k2 && a.v2 && a.ldk2 % 8 == 0 && a.ldv2 % 8 == 0, "attention: dual source needs k2 / v2");
    if ((rc = make_qkv_tmap(&tk2, a.k2, a.B, a.Lk2, a.H, a.ldk2))) return rc;
    if ((rc = make_qkv_tmap(&tv2, a.v2, a.B, a.Lk2, a.H, a.ldv2))) return rc;
  } else {
    tk2 = tk;
    tv2 = tv;
  }
  CE_ENSURE_SMEM(attention_fwd_kernel, SmemLayout::total);
  dim3 grid((a.Lq + BQ - 1) / BQ, a.H, a.B);
  attention_fwd_kernel<<<grid, ATTN_THREADS, SmemLayout::total, stream>>>(tq, tk, tv, tk2, tv2, a);
  CE_CHECK_CUDA(cudaGetLastError());
  return CE_OK;
}

}  // namespace ce
