// feas.cu — K1: the dense pods x templates Filter pass (SchedulablePodGroups for EVERY pending pod,
// core/scaleup/orchestrator/orchestrator.go:603-638 -> RunFiltersOnNode, plugin_runner.go:131).
//
// thread = pod.  NodeResourcesFit (noderesources/fit.go:649-736) is `request_r > free_r` for every
// requested resource; the int64 operands are order-preserving dictionary encoded at load time:
//     rank_req(v)  = 1-based index of v among the sorted distinct positive requests of that resource
//                    (0 when the pod does not request it: such a resource is never checked, fit.go:670-704)
//     rank_free(f) = number of distinct request values <= f
//     request > free  <=>  rank_req > rank_free            (exact, both directions)
//
// LUT variant (default): the ranks are small dictionaries, so "rank_req <= rank_free" for 32 templates is
// ONE word of a threshold bitmap indexed by (dim, rank_req):
//     lut[base_a + k][tw] bit j = (k <= rank_free_a(template tw*32+j))
// A pod's verdict word is the AND of A shared-memory words and its two class words (pre_ok / post_ok of
// the size-independent plugins, read with 128-bit loads through L1: neighbouring pods share classes).
// Rows are staged with an odd pitch so that lanes reading different rows hit different banks.
//
// Bit-sliced variant (fallback when the threshold rows do not fit in shared memory, CAE_K1_BITSLICE=1):
// the template ranks are stored bit-sliced (slice b, word tw = bit b of the ranks of templates tw*32..+31)
// and a lane compares its pod against 32 templates with the MSB-first bit-serial comparator
// (gt |= eq & r & ~f; eq &= ~(r ^ f)).
//
// Both: a 5-stage shuffle transpose of the warp's 32x32 verdict block yields the template-major words of
// the output bit matrix; they are flushed in runs of consecutive words per template row and pop-counted into
// the fit histogram.  The histogram accumulators clean themselves: the last thread block of a template
// chunk publishes fit_count and zeroes the accumulator, so a step is ONE kernel launch (no memset).
#include <algorithm>
#include <climits>

#include "engine.h"

namespace cae {

struct LutLayout {
  int A, rows;               // active dims, threshold rows (all dims)
  int base[CAE_MAX_RES];
  uint32_t mask[CAE_MAX_RES];
  uint8_t word[CAE_MAX_RES], shift[CAE_MAX_RES];
};

static LutLayout lut_layout(const Engine* e) {
  LutLayout lay{};
  lay.A = e->A;
  lay.rows = e->lut_rows;
  for (int d = 0; d < e->A; ++d) {
    lay.base[d] = e->lut_base[d]; lay.mask[d] = e->lut_mask[d]; lay.word[d] = e->lut_word[d]; lay.shift[d] = e->lut_shift[d];
  }
  return lay;
}

// per pending pod of this rank's shard: packed request ranks (bit-sliced variant), the threshold-row id of every
// active dim (LUT variant: base_a + rank_req_a, 0xFFFF when the rows do not fit 16 bits) and the two class ids
__global__ void expand_pods_kernel(const int32_t* __restrict__ pend_spec, int p_begin, int Pl, int W, LutLayout lay,
                                   const uint32_t* __restrict__ spec_w, const int32_t* __restrict__ spec_sc,
                                   const int32_t* __restrict__ spec_dc, uint32_t* __restrict__ pod_w,
                                   uint16_t* __restrict__ pod_row, int32_t* __restrict__ pod_sc, int32_t* __restrict__ pod_dc) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Pl) return;
  int spec = pend_spec[p_begin + p];
  for (int w = 0; w < W; ++w) pod_w[(size_t)w * Pl + p] = spec_w[(size_t)spec * FEAS_MAX_W + w];
  for (int d = 0; d < lay.A; ++d) {
    const int row = lay.base[d] + (int)((spec_w[(size_t)spec * FEAS_MAX_W + lay.word[d]] >> lay.shift[d]) & lay.mask[d]);
    pod_row[(size_t)d * Pl + p] = (uint16_t)min(row, 0xFFFF);
  }
  pod_sc[p] = spec_sc[spec];
  pod_dc[p] = spec_dc[spec];
}

int launch_expand_pods(Engine* e) {
  if (e->Pl == 0) return 0;
  expand_pods_kernel<<<(e->Pl + 255) / 256, 256, 0, e->stream>>>(e->dobj.pend_spec, e->p_begin, e->Pl, e->W, lut_layout(e), e->d_spec_w,
                                                                   e->d_spec_sc, e->d_spec_dc, e->d_pod_w, e->d_pod_row, e->d_pod_sc, e->d_pod_dc);
  e->stats.kernel_launches++;
  CAE_KERNEL_OK();
  return 0;
}

constexpr int K1_TW = FEAS_TW;            // template words (x32 templates) per thread block
constexpr int K1_TCHUNK = K1_TW * 32;
constexpr int K1_LPITCH = K1_TW + 1;      // odd row pitch of the staged threshold rows

// Fused exchange of the fit histogram over peer memory (see cae_peer_attach in include/caengine.h): an
// all-gather.  Every rank owns an exchange buffer [2 parities][PEER_MAX ranks][PEER_CAP] of (count, step tag) slots; a
// step writes the local histogram into row `rank` of EVERY rank's buffer — one 8-byte store per template over NVLink —
// and reads the rows of its own buffer until every slot carries this step's tag (k1_finish below).
struct PeerPush {
  int world, rank;           // world 0 = disabled
  int tag;                   // step number carried by every slot of this step (never 0)
  int2* data[8];             // every rank's [PEER_MAX][PEER_CAP] block of (count, tag) slots of this step's parity (P2P-mapped)
  const int2* self;          // data[rank]
  int32_t* done_ctr;         // local: template chunks published
  int32_t* status;           // local: set to 1 when a peer never arrived
};

struct K1Args {
  int Pl, Plw, T, Tw, Twp, N, U, W;
  int G, gq, gr;                          // thread blocks per template chunk; block x takes gq (+1 if x < gr) pod words
  const uint32_t* pod_w;
  const uint16_t* pod_row;                // [A][Pl] threshold-row ids
  const int32_t *pod_sc, *pod_dc;
  const uint32_t *tslice, *rlut;
  const int32_t* tmpl_slots;
  const uint32_t *pre_ok, *post_ok;       // [classes][Twp]
  const uint8_t *pre_code, *post_code;
  uint32_t* fit_bits;
  int32_t *fit_count, *fit_acc, *chunk_done;
  uint8_t* reasons;
};

__device__ __forceinline__ int k1_ld_acquire_sys(const int32_t* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void k1_red_release_sys(int32_t* p, int v) {
  asm volatile("red.release.sys.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void k1_st_volatile_v2(int2* p, int x, int y) {
  asm volatile("st.volatile.global.v2.s32 [%0], {%1, %2};" ::"l"(p), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ int2 k1_ld_volatile_v2(const int2* p) {
  int2 v;
  asm volatile("ld.volatile.global.v2.s32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long k1_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Phase timeline of the dense pass, compiled in only with -DCAE_K1_PROF (scripts/k1_floor.py reads it through
// cae_k1_prof_read): k1_prof[0] = %globaltimer when the stream reached the launch (a one-thread kernel queued just
// before it), then per thread block K1_PROF_STAMPS stamps taken by thread 0: entry, loads done, compute done,
// bit-matrix stores issued, exit.
#ifdef CAE_K1_PROF
constexpr int K1_PROF_MAX_BLOCKS = 8192, K1_PROF_STAMPS = 5;
__device__ unsigned long long k1_prof[1 + K1_PROF_STAMPS * K1_PROF_MAX_BLOCKS];
#define K1_STAMP(i)                                                                                 \
  do {                                                                                              \
    const int b_ = blockIdx.y * gridDim.x + blockIdx.x;                                             \
    if (threadIdx.x == 0 && b_ < K1_PROF_MAX_BLOCKS) k1_prof[1 + K1_PROF_STAMPS * b_ + (i)] = k1_globaltimer(); \
  } while (0)
__global__ void k1_prof_mark_kernel() { k1_prof[0] = k1_globaltimer(); }
#else
#define K1_STAMP(i) do {} while (0)
#endif

// ---- epilogue shared by both variants -------------------------------------------------------------------
// s_cnt holds this block's counts for templates t0 .. t0+K1_TCHUNK.  The LAST block of the chunk to arrive
// publishes fit_count = accumulator and zeroes the accumulator for the next launch.  With a peer exchange
// attached, the last CHUNK to be published adds the whole local histogram into every rank's exchange buffer
// over NVLink (system-scope atomics on peer memory) and signals arrival.
__device__ __forceinline__ void k1_finish(const K1Args& a, const PeerPush& pp, const int32_t* s_cnt, int t0, int tid, int nthreads) {
  __shared__ int s_flag;
  for (int i = tid; i < K1_TCHUNK; i += nthreads) {
    const int c = s_cnt[i];
    if (c && t0 + i < a.T) atomicAdd(&a.fit_acc[t0 + i], c);
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_flag = atomicAdd(&a.chunk_done[blockIdx.y], 1) == (int)gridDim.x - 1;
  }
  __syncthreads();
  if (!s_flag) return;
  __threadfence();
  for (int i = tid; i < K1_TCHUNK; i += nthreads) {
    const int t = t0 + i;
    if (t < a.T) {
      a.fit_count[t] = __ldcg(&a.fit_acc[t]);
      a.fit_acc[t] = 0;
    }
  }
  if (tid == 0) a.chunk_done[blockIdx.y] = 0;
  if (!pp.world) return;
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_flag = atomicAdd(pp.done_ctr, 1) == (int)gridDim.y - 1;
  }
  __syncthreads();
  if (!s_flag) return;
  // The block that published the LAST chunk owns the complete local histogram: all-gather it with a low-latency protocol
  // (the one NCCL calls LL): every slot is ONE 8-byte store of (count, step tag) into the peer's buffer over NVLink, so a
  // reader that sees this step's tag in a slot has this step's count — no fence, no separate flag, no round trip waiting
  // for acknowledgements.  Two parities alternate: a rank can only write step s+2 after it has READ every peer's step s+1,
  // which that peer wrote after it finished reading step s.
  __threadfence();
  const int tag = pp.tag;
  // data[] is only indexed by unrolled constants and data[rank] comes as `self`: a run-time index would make every
  // launch copy the whole struct to local memory, also at N = 1
#pragma unroll
  for (int r = 0; r < Engine::PEER_MAX; ++r) {
    if (r < pp.world) {
      int2* dst = pp.data[r] + (size_t)pp.rank * Engine::PEER_CAP;
      for (int t = tid; t < a.T; t += nthreads) k1_st_volatile_v2(dst + t, __ldcg(&a.fit_count[t]), tag);
    }
  }
  const int2* mine = pp.self;
  const unsigned long long t0ns = k1_globaltimer();
  int ok = 1;
  for (int t = tid; t < a.T && ok; t += nthreads) {
    // all ranks' slots of this template in flight at once (independent loads), then only the late ones are polled again
    int2 x[Engine::PEER_MAX];
    unsigned pending = 0;
#pragma unroll
    for (int r = 0; r < Engine::PEER_MAX; ++r)
      if (r < pp.world) x[r] = k1_ld_volatile_v2(mine + (size_t)r * Engine::PEER_CAP + t);
#pragma unroll
    for (int r = 0; r < Engine::PEER_MAX; ++r)
      if (r < pp.world && x[r].y != tag) pending |= 1u << r;
    for (int spins = 0; pending; ) {
#pragma unroll
      for (int r = 0; r < Engine::PEER_MAX; ++r)
        if ((pending >> r) & 1u) {
          x[r] = k1_ld_volatile_v2(mine + (size_t)r * Engine::PEER_CAP + t);
          if (x[r].y == tag) pending &= ~(1u << r);
        }
      if (pending && (++spins & 1023) == 0 && k1_globaltimer() - t0ns > 2000000000ull) { ok = 0; break; }   // 2 s: a peer died; fail, never hang
    }
    int v = 0;
#pragma unroll
    for (int r = 0; r < Engine::PEER_MAX; ++r)
      if (r < pp.world) v += x[r].x;
    if (ok) a.fit_count[t] = v;
  }
  if (!ok) atomicExch(pp.status, 1);
  if (tid == 0) *pp.done_ctr = 0;
}

// ---- 32x32 bit transposes across a warp ---------------------------------------------------------------------
// lane i holds row i of a 32x32 bit matrix; afterwards lane j holds column j (bit i = M[i][j]).
// Stages 16 and 8 move whole bytes: one shuffle + one byte permute.  Stages 4, 2, 1: the sender rotates the
// part the partner needs into place (funnel shift), the receiver merges under a per-lane mask (one LOP3).
struct TransposeConsts { uint32_t sel16, sel8, amt[3], keep[3]; };

__device__ __forceinline__ uint32_t opaque(uint32_t v) {   // keep a per-lane constant in a register instead of re-deriving it
  uint32_t r;
  asm volatile("mov.b32 %0, %1;" : "=r"(r) : "r"(v));
  return r;
}

__device__ __forceinline__ TransposeConsts transpose_consts(int lane) {
  TransposeConsts c;
  c.sel16 = opaque((lane & 16) ? 0x3276u : 0x5410u);
  c.sel8 = opaque((lane & 8) ? 0x3715u : 0x6240u);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int s = 4 >> i;
    const uint32_t lowmask = s == 4 ? 0x0F0F0F0Fu : s == 2 ? 0x33333333u : 0x55555555u;
    c.amt[i] = opaque((lane & s) ? (uint32_t)s : (uint32_t)(32 - s));   // set lanes send their low part up, clear lanes their high part down
    c.keep[i] = opaque((lane & s) ? ~lowmask : lowmask);
  }
  return c;
}

__device__ __forceinline__ uint32_t bitselect(uint32_t x, uint32_t y, uint32_t keep) {   // keep ? x : y, bitwise
  uint32_t r;
  asm("lop3.b32 %0, %1, %2, %3, 0xE4;" : "=r"(r) : "r"(x), "r"(y), "r"(keep));
  return r;
}

// two independent blocks at once: twice the instruction-level parallelism on the shuffle latency
__device__ __forceinline__ void warp_transpose32x2(uint32_t& a, uint32_t& b, const TransposeConsts& c) {
  uint32_t ya = __shfl_xor_sync(0xffffffffu, a, 16), yb = __shfl_xor_sync(0xffffffffu, b, 16);
  a = __byte_perm(a, ya, c.sel16);
  b = __byte_perm(b, yb, c.sel16);
  ya = __shfl_xor_sync(0xffffffffu, a, 8);
  yb = __shfl_xor_sync(0xffffffffu, b, 8);
  a = __byte_perm(a, ya, c.sel8);
  b = __byte_perm(b, yb, c.sel8);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    ya = __shfl_xor_sync(0xffffffffu, __funnelshift_l(a, a, c.amt[i]), 4 >> i);
    yb = __shfl_xor_sync(0xffffffffu, __funnelshift_l(b, b, c.amt[i]), 4 >> i);
    a = bitselect(a, ya, c.keep[i]);
    b = bitselect(b, yb, c.keep[i]);
  }
}

__device__ __forceinline__ uint32_t warp_transpose32(uint32_t x, int lane) {
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) {
    const uint32_t lowmask = s == 16 ? 0x0000FFFFu : s == 8 ? 0x00FF00FFu : s == 4 ? 0x0F0F0F0Fu : s == 2 ? 0x33333333u : 0x55555555u;
    const uint32_t y = __shfl_xor_sync(0xffffffffu, x, s);
    x = (lane & s) ? ((x & ~lowmask) | ((y & ~lowmask) >> s)) : ((x & lowmask) | ((y & lowmask) << s));
  }
  return x;
}

// ---- LUT variant --------------------------------------------------------------------------------------------
// Resident warps per SM the kernel is compiled for, the most that keeps it free of spills: 48 (at most 40 registers per
// thread), 32 (64 registers) for the dim counts that would spill at 40, 16 for the reasons variant (its per-template
// loop of byte stores is bound by memory, not by the warps in flight).
template <int A, bool REASONS>
constexpr int k1_lut_warps_per_sm() { return REASONS ? 16 : (A == 0 || A > 5) ? 32 : 48; }

template <int A, bool REASONS, int NW>
__global__ void __launch_bounds__(NW * 32, k1_lut_warps_per_sm<A, REASONS>() / NW)
feasibility_lut_kernel(K1Args a, int rows, PeerPush pp) {
  extern __shared__ uint32_t k1_smem[];
  constexpr int NT = NW * 32;
  constexpr int PAD = K1_TCHUNK + 32 / NW;                     // flush reads (wv, tl) hit 32 distinct banks
  uint32_t* s_lut = k1_smem;                                   // [rows][K1_LPITCH]
  uint32_t* s_out = s_lut + (size_t)max(rows, 1) * K1_LPITCH;       // [NW][PAD]
  int32_t* s_cnt = reinterpret_cast<int32_t*>(s_out + NW * PAD);    // [K1_TCHUNK]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tw0 = blockIdx.y * K1_TW;
  const int t0 = tw0 * 32;
  // this block's run of pod words (an even split of Plw over the G blocks of the chunk; 1..NW words)
  const int pwb = (int)blockIdx.x * a.gq + min((int)blockIdx.x, a.gr);
  const int npw = a.gq + ((int)blockIdx.x < a.gr ? 1 : 0);
  const int p = (pwb + warp) * 32 + lane;
  const bool valid = warp < npw && p < a.Pl;
  K1_STAMP(0);

#pragma unroll 1
  for (int i = tid; i < rows * K1_TW; i += NT) {
    const int row = i / K1_TW, w = i % K1_TW;
    s_lut[row * K1_LPITCH + w] = a.rlut[(size_t)row * a.Twp + tw0 + w];   // pitch padded to whole chunks: always in bounds
  }
  for (int i = tid; i < K1_TCHUNK; i += NT) s_cnt[i] = 0;

  int off[A > 0 ? A : 1];
#pragma unroll
  for (int d = 0; d < A; ++d) off[d] = valid ? (int)a.pod_row[(size_t)d * a.Pl + p] * K1_LPITCH : 0;
  const int sc = valid ? a.pod_sc[p] : 0;
  const int dc = valid ? a.pod_dc[p] : 0;
  // class words of this pod for the chunk's K1_TW template words (rows are 64 B aligned: 128-bit loads)
  uint32_t cls[K1_TW];
  {
    const uint4* pre = reinterpret_cast<const uint4*>(a.pre_ok + (size_t)sc * a.Twp + tw0);
    const uint4* post = reinterpret_cast<const uint4*>(a.post_ok + (size_t)dc * a.Twp + tw0);
#pragma unroll
    for (int q = 0; q < K1_TW / 4; ++q) {
      uint4 u = make_uint4(0, 0, 0, 0);
      if (valid) {
        const uint4 x = __ldg(pre + q), y = __ldg(post + q);
        u = make_uint4(x.x & y.x, x.y & y.y, x.z & y.z, x.w & y.w);
      }
      cls[4 * q + 0] = u.x; cls[4 * q + 1] = u.y; cls[4 * q + 2] = u.z; cls[4 * q + 3] = u.w;
    }
  }
  const TransposeConsts tc = transpose_consts(lane);
  __syncthreads();
  K1_STAMP(1);

#pragma unroll
  for (int tw = 0; tw < K1_TW; tw += 2) {
    uint32_t fit0 = 0xffffffffu, fit1 = 0xffffffffu;
#pragma unroll
    for (int d = 0; d < A; ++d) {
      fit0 &= s_lut[off[d] + tw];
      fit1 &= s_lut[off[d] + tw + 1];
    }
    if (REASONS) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int wglob = tw0 + tw + h;
        const uint32_t fit = h ? fit1 : fit0;
        if (valid && wglob < a.Tw) {
          for (int j = 0; j < 32; ++j) {
            const int t = wglob * 32 + j;
            if (t >= a.T) break;
            // first failing plugin in Filter order: static plugins, NodeResourcesFit, then PTS / IPA
            uint8_t rs = a.pre_code[(size_t)sc * a.U + a.N + t] & 0x0F;
            if (rs == 0) rs = (!((fit >> j) & 1u) || a.tmpl_slots[t] < 1) ? CAE_R_FIT : a.post_code[(size_t)dc * a.T + t];
            a.reasons[(size_t)t * a.Pl + p] = rs;
          }
        }
      }
    }
    uint32_t c0 = fit0 & cls[tw], c1 = fit1 & cls[tw + 1];
    warp_transpose32x2(c0, c1, tc);      // words of templates t0 + tw*32 + lane (and + 32) over this warp's pods
    s_out[warp * PAD + tw * 32 + lane] = c0;
    s_out[warp * PAD + (tw + 1) * 32 + lane] = c1;
    atomicAdd(&s_cnt[tw * 32 + lane], __popc(c0));
    atomicAdd(&s_cnt[(tw + 1) * 32 + lane], __popc(c1));
  }
  __syncthreads();
  K1_STAMP(2);
  // flush: NW consecutive threads write the block's run of pod words of one template row
  if (a.fit_bits) {
    const int wv = tid % NW;
    if (wv < npw) {
      uint32_t* dst = a.fit_bits + (size_t)(t0 + tid / NW) * a.Plw + pwb + wv;
      const uint32_t* src = s_out + wv * PAD + tid / NW;
      const size_t stride = (size_t)32 * a.Plw;
      const int kmax = min(K1_TCHUNK / 32, (a.T - t0 - tid / NW + 31) / 32);   // rows t0 + tid/NW + 32k < T
#pragma unroll 4
      for (int k = 0; k < kmax; ++k, dst += stride, src += 32) *dst = *src;
    }
  }
  K1_STAMP(3);
  k1_finish(a, pp, s_cnt, t0, tid, NT);
  K1_STAMP(4);
}

// ---- bit-sliced variant ---------------------------------------------------------------------------------------
constexpr int K1_THREADS = 256;
constexpr int K1_WARPS = K1_THREADS / 32;
constexpr int K1_PAD = K1_TCHUNK + 4;

struct FeasLayout {
  uint32_t fstart;           // bit b: slice b starts a field
  int nb;                    // real slices (the rest is zero padding)
  uint8_t sword[32], sshift[32];
};

template <int B, bool REASONS>
__global__ void __launch_bounds__(K1_THREADS)
feasibility_kernel(K1Args a, FeasLayout lay, PeerPush pp) {
  __shared__ uint32_t s_sl[B > 0 ? B : 1][K1_TW];
  __shared__ uint32_t s_out[K1_WARPS][K1_PAD];
  __shared__ int32_t s_cnt[K1_TCHUNK];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int p = blockIdx.x * K1_THREADS + tid;
  const int tw0 = blockIdx.y * K1_TW;
  const int t0 = tw0 * 32;

  for (int i = tid; i < B * K1_TW; i += K1_THREADS) {
    const int b = i / K1_TW, w = i % K1_TW;
    s_sl[b][w] = (tw0 + w < a.Tw) ? a.tslice[(size_t)b * a.Tw + tw0 + w] : 0u;
  }
  for (int i = tid; i < K1_TCHUNK; i += K1_THREADS) s_cnt[i] = 0;
  const bool valid = p < a.Pl;
  // the pod's rank bits as all-ones / all-zeros masks, one register per slice
  uint32_t r[B > 0 ? B : 1];
  {
    uint32_t pw[FEAS_MAX_W];
#pragma unroll
    for (int w = 0; w < FEAS_MAX_W; ++w) pw[w] = (valid && w < a.W) ? a.pod_w[(size_t)w * a.Pl + p] : 0u;
#pragma unroll
    for (int b = 0; b < B; ++b) {
      const uint32_t word = lay.sword[b] == 0 ? pw[0] : lay.sword[b] == 1 ? pw[1] : lay.sword[b] == 2 ? pw[2] : pw[3];
      r[b] = b < lay.nb ? 0u - ((word >> lay.sshift[b]) & 1u) : 0u;
    }
  }
  const int sc = valid ? a.pod_sc[p] : 0;
  const int dc = valid ? a.pod_dc[p] : 0;
  __syncthreads();

#pragma unroll 1
  for (int tw = 0; tw < K1_TW; ++tw) {
    const int wglob = tw0 + tw;
    uint32_t row = 0;
    if (wglob < a.Tw) {
      // bit-serial "rank_req > rank_free" for 32 templates at once; fields concatenated, MSB first
      uint32_t gt = 0, eq = 0;
#pragma unroll
      for (int b = 0; b < B; ++b) {
        const uint32_t f = s_sl[b][tw];
        if ((lay.fstart >> b) & 1u) eq = 0xffffffffu;  // uniform: a new field starts
        gt |= eq & r[b] & ~f;
        eq &= ~(r[b] ^ f);
      }
      row = valid ? (~gt & a.pre_ok[(size_t)sc * a.Twp + wglob] & a.post_ok[(size_t)dc * a.Twp + wglob]) : 0u;
      if (REASONS) {
        if (valid) {
          for (int j = 0; j < 32; ++j) {
            const int t = wglob * 32 + j;
            if (t >= a.T) break;
            uint8_t rs = a.pre_code[(size_t)sc * a.U + a.N + t] & 0x0F;
            if (rs == 0) rs = (((gt >> j) & 1u) || a.tmpl_slots[t] < 1) ? CAE_R_FIT : a.post_code[(size_t)dc * a.T + t];
            a.reasons[(size_t)t * a.Pl + p] = rs;
          }
        }
      }
    }
    const uint32_t col = warp_transpose32(row, lane);  // word of template t0 + tw*32 + lane over this warp's pods
    s_out[warp][tw * 32 + lane] = col;
    if (col) atomicAdd(&s_cnt[tw * 32 + lane], __popc(col));
  }
  __syncthreads();
  // flush: 8 consecutive words (one 32 B sector) per template row
  const int pw0 = blockIdx.x * K1_WARPS;
  for (int i = tid; i < K1_TCHUNK * K1_WARPS; i += K1_THREADS) {
    const int tl = i / K1_WARPS, wv = i % K1_WARPS;
    const int t = t0 + tl;
    if (t < a.T && pw0 + wv < a.Plw && a.fit_bits) a.fit_bits[(size_t)t * a.Plw + pw0 + wv] = s_out[wv][tl];
  }
  k1_finish(a, pp, s_cnt, t0, tid, K1_THREADS);
}

// ---- launch ----------------------------------------------------------------------------------------------------
static PeerPush peer_push_args(Engine* e) {
  PeerPush pp{};
  if (e->peer_world > 1 && e->T <= Engine::PEER_CAP) {
    const int par = (int)(e->peer_step & 1);
    const size_t blk = (size_t)Engine::PEER_MAX * Engine::PEER_CAP;   // slots per parity
    pp.world = e->peer_world;
    pp.rank = e->cfg.rank;
    e->peer_step += 1;
    pp.tag = (int)(e->peer_step & 0x7fffffff);
    if (pp.tag == 0) pp.tag = 1;
    for (int r = 0; r < e->peer_world; ++r) pp.data[r] = reinterpret_cast<int2*>(e->peer_base[r]) + par * blk;
    pp.self = pp.data[pp.rank];
    pp.done_ctr = e->d_xbuf + 4 * blk + 8;
    pp.status = e->d_xbuf + 4 * blk + 9;
  }
  return pp;
}

static K1Args k1_args(Engine* e) {
  K1Args a{};
  a.Pl = e->Pl; a.Plw = e->Plw; a.T = e->T; a.Tw = e->Tw; a.Twp = e->Twp; a.N = e->N; a.U = e->U; a.W = e->W;
  a.G = 1;
  a.pod_w = e->d_pod_w; a.pod_row = e->d_pod_row; a.pod_sc = e->d_pod_sc; a.pod_dc = e->d_pod_dc;
  a.tslice = e->d_tslice; a.rlut = e->d_rlut; a.tmpl_slots = e->d_tmpl_slots;
  a.pre_ok = e->d_pre_ok; a.post_ok = e->d_post_ok; a.pre_code = e->d_pre_code; a.post_code = e->d_post_code;
  a.fit_bits = e->d_fit_bits; a.fit_count = e->d_fit_count; a.fit_acc = e->d_fit_acc; a.chunk_done = e->d_chunk_done;
  a.reasons = e->d_reasons;
  return a;
}

template <int B>
static void launch_feas_b(Engine* e, bool want_reasons, K1Args a, const PeerPush& pp) {
  dim3 grid((e->Pl + K1_THREADS - 1) / K1_THREADS, e->Twp / K1_TW);
  FeasLayout lay;
  lay.fstart = e->feas_fstart;
  lay.nb = e->feas_B;
  for (int b = 0; b < 32; ++b) { lay.sword[b] = e->feas_sword[b]; lay.sshift[b] = e->feas_sshift[b]; }
  if (want_reasons) feasibility_kernel<B, true><<<grid, K1_THREADS, 0, e->stream>>>(a, lay, pp);
  else feasibility_kernel<B, false><<<grid, K1_THREADS, 0, e->stream>>>(a, lay, pp);
}

template <int A, bool REASONS, int NW>
static int launch_feas_lut_arw(Engine* e, K1Args a, const PeerPush& pp) {
  const int chunks = e->Twp / K1_TW;
  // one wave when it fits: the pod words are split evenly over as many blocks as the SMs hold at once
  const int slots = e->sm_count * (k1_lut_warps_per_sm<A, REASONS>() / NW);
  const int g_min = (e->Plw + NW - 1) / NW;
  a.G = std::max(g_min, std::min(e->Plw, std::max(1, slots / chunks)));
  a.gq = e->Plw / a.G;
  a.gr = e->Plw % a.G;
  dim3 grid(a.G, chunks);
  const size_t smem = sizeof(uint32_t) * ((size_t)std::max(e->lut_rows, 1) * K1_LPITCH + NW * (K1_TCHUNK + 32 / NW) + K1_TCHUNK);
  auto kern = feasibility_lut_kernel<A, REASONS, NW>;
  if (smem > 48 * 1024) CAE_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<grid, NW * 32, smem, e->stream>>>(a, e->lut_rows, pp);
  return 0;
}

template <int A>
static int launch_feas_lut_a(Engine* e, bool want_reasons, const K1Args& a, const PeerPush& pp) {
  return want_reasons ? launch_feas_lut_arw<A, true, 16>(e, a, pp) : launch_feas_lut_arw<A, false, 16>(e, a, pp);
}

constexpr int K1_LUT_MAX_ROWS = FEAS_LUT_MAX_ROWS;

int launch_feasibility(Engine* e, bool want_reasons) {
  if (e->Tw == 0) return 0;
  if (e->Pl == 0) {   // no pending pods on this rank: an all-zero histogram (the exchange, if any, is the caller's NCCL path)
    CAE_CUDA(cudaMemsetAsync(e->d_fit_count, 0, sizeof(int32_t) * e->T, e->stream));
    return 0;
  }
  if (e->peer_world > 1 && e->T > Engine::PEER_CAP) {   // never hand back a local histogram as if it were the global one
    set_error("fused histogram exchange: more templates than the exchange buffer holds (use the NCCL all-reduce of cae_device_buffer(0))");
    return 1;
  }
#ifdef CAE_K1_PROF
  {
    void* prof = nullptr;
    CAE_CUDA(cudaGetSymbolAddress(&prof, k1_prof));
    CAE_CUDA(cudaMemsetAsync(prof, 0, sizeof(k1_prof), e->stream));
    k1_prof_mark_kernel<<<1, 1, 0, e->stream>>>();
  }
#endif
  const PeerPush pp = peer_push_args(e);
  const K1Args a = k1_args(e);
  if (!e->force_bitslice && e->lut_rows <= K1_LUT_MAX_ROWS) {
    int rc = 0;
    switch (e->A) {
      case 0: rc = launch_feas_lut_a<0>(e, want_reasons, a, pp); break;
      case 1: rc = launch_feas_lut_a<1>(e, want_reasons, a, pp); break;
      case 2: rc = launch_feas_lut_a<2>(e, want_reasons, a, pp); break;
      case 3: rc = launch_feas_lut_a<3>(e, want_reasons, a, pp); break;
      case 4: rc = launch_feas_lut_a<4>(e, want_reasons, a, pp); break;
      case 5: rc = launch_feas_lut_a<5>(e, want_reasons, a, pp); break;
      case 6: rc = launch_feas_lut_a<6>(e, want_reasons, a, pp); break;
      case 7: rc = launch_feas_lut_a<7>(e, want_reasons, a, pp); break;
      default: rc = launch_feas_lut_a<8>(e, want_reasons, a, pp); break;
    }
    if (rc) return rc;
  } else {
    // slices beyond feas_B are all-zero with r = 0: they change nothing (padding to a multiple of 4)
    const int Bp = e->feas_B == 0 ? 0 : (e->feas_B + 3) / 4 * 4;
    switch (Bp) {
      case 0: launch_feas_b<0>(e, want_reasons, a, pp); break;
      case 4: launch_feas_b<4>(e, want_reasons, a, pp); break;
      case 8: launch_feas_b<8>(e, want_reasons, a, pp); break;
      case 12: launch_feas_b<12>(e, want_reasons, a, pp); break;
      case 16: launch_feas_b<16>(e, want_reasons, a, pp); break;
      case 20: launch_feas_b<20>(e, want_reasons, a, pp); break;
      case 24: launch_feas_b<24>(e, want_reasons, a, pp); break;
      case 28: launch_feas_b<28>(e, want_reasons, a, pp); break;
      default: launch_feas_b<32>(e, want_reasons, a, pp); break;
    }
  }
  e->stats.kernel_launches++;
  CAE_KERNEL_OK();
  return 0;
}

}  // namespace cae

#ifdef CAE_K1_PROF
// the phase stamps of the last dense pass (synchronous): 1 + K1_PROF_STAMPS * blocks values, returns the count copied
extern "C" int cae_k1_prof_read(unsigned long long* out, int n) {
  n = std::max(0, std::min(n, 1 + cae::K1_PROF_STAMPS * cae::K1_PROF_MAX_BLOCKS));
  if (cudaMemcpyFromSymbol(out, cae::k1_prof, sizeof(unsigned long long) * n) != cudaSuccess) return -1;
  return n;
}
#endif
