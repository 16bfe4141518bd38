// MusicGen LM decode step as ONE persistent kernel (sm_90a): every layer of LMModel.forward on one token per row
// (audiocraft/models/lm.py:221-268, modules/transformer.py:550-574, 693-713) runs inside a single cooperative launch of
// one CTA per SM; the CFG mix + sampler (lm.cu: lm_sample_kernel) follows as the second and last kernel of the step.
//
// Why one kernel.  A decode step is a strict chain of ~12 small dependent phases per layer.  As separate kernels each
// phase pays a launch boundary that is long against the 0.1-0.3 us its HBM traffic needs.
// Here the phases are separated by a grid barrier (csrc/gridbar.cuh, < 1 us) and, because weights are static, a
// dedicated producer warp streams them with TMA bulk copies through a deep shared-memory ring that runs AHEAD of the
// phase the compute warps are in: the HBM weight stream never stops at a phase boundary.
//
// Work decomposition.  Every GEMM y[rows][N] = act[rows][K] . W[N][K]^T is cut into items = (128-feature tile, K slice)
// so that ~all SMs hold one item; the 128 x 64 fp16 weight tiles are pre-packed (acb_lm_pack_weight) in the
// canonical 128-byte-swizzled K-major layout, so a tile is ONE contiguous 16 KB bulk copy and is consumed straight from shared
// memory by wgmma (swap-AB: features on M = 2 x 64, one warpgroup each, rows on N = R in {16,32,48,64}).  No thread ever
// touches a weight fragment.  Items write fp32 partial sums; the consumer of a GEMM reduces them in a fixed order
// (bit-reproducible): attention sums the 4 QKV partials of its head, the residual phases sum the O / FFN2 partials
// into x and emit LayerNorm statistics per d/8 columns, so the next GEMM normalises its activations while it stages them.
//
// Phases per layer (grid barrier after each):
//   QKV gemm (LN1 on load) | self-attention (+KV append) | O gemm | residual+stats |
//   CQ gemm (LNc on load) | cross-attention | CO gemm | residual+stats | FF1 gemm (LN2 on load) | gelu+reduce |
//   FF2 gemm | residual+stats          then: heads gemm (out_norm on load) | logits reduce.
#include "lm_step.cuh"
#include "gridbar.cuh"
#include "wgmma.cuh"
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

namespace {

// CODE SIZE IS A FIRST-ORDER COST HERE.  Every SM executes each phase's code once per layer, ~0.5 ms apart per phase kind
// at best: what does not fit the instruction cache is fetched from L2 like data (a first version with wide predicated unrolls
// and phases inlined at every call site had every phase several times slower than its memory traffic explains).  Hence: phases are __noinline__ functions
// shared by all their call sites, loops are rolled or unrolled by <= 4, and memory-level parallelism comes from 16 compute
// warps per CTA instead of from unrolling.
constexpr int NCW = 8;                  // compute warps = two warpgroups, one per 64-feature half of a weight tile
constexpr int CT = NCW * 32;            // compute threads
constexpr int BLOCK = CT + 32;          // + the TMA producer warp
constexpr int TILE_BYTES = 16384;       // 128 features x 64 K, fp16
constexpr int TILE_HALVES = 8192;
constexpr int MAX_STAGE = 14;
constexpr int SCRATCH_BYTES = 12288;
static_assert((2 * NCW + 2 * 3 * NCW + 3 * NCW * 64 + 3 * 192) * 4 + 512 <= SCRATCH_BYTES, "scratch does not fit");     // mbarriers + small per-phase scratch behind the ring and the activation tile
// The grid-barrier poller lives in warp 1, not on the scheduler of the producer warp (id NCW, scheduler NCW % 4 = 0).
constexpr int ISSUE_WARP = 1;
constexpr int NACC = 4;                 // independent accumulator chains per GEMM item (K steps rotate over them)
constexpr int ATT_GROUP = 3;            // self-attention tasks a CTA stages / merges together (one barrier pair per group)
constexpr int ATT_UNROLL = 4;           // positions-groups per batch and lane; two batches are live (software pipeline)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok = 0;
    do {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!ok);
}
// A warp that SPINS on a barrier steals issue slots from the other warps of its scheduler.  Waiters that may wait long
// (the producer on a full ring) therefore sleep between polls, and during a grid barrier everybody but one warp blocks on
// a hardware barrier (bar.sync) instead of polling.
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity, unsigned ns) {
    uint32_t ok = 0;
    for (;;) {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
        if (ok) break;
        __nanosleep(ns);
    }
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// barrier among the compute warps only (the producer warp never joins)
__device__ __forceinline__ void cbar() { asm volatile("bar.sync 1, %0;" ::"n"(CT) : "memory"); }

__device__ __forceinline__ float half_round(float v) { return __half2float(__float2half_rn(v)); }
__device__ __forceinline__ float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

struct Smem {
    unsigned char* ring; unsigned char* act;
    uint64_t* full; uint64_t* empty;
    float* red;                     // [2][NCW]
    float* wm; float* wl; float* wacc;   // attention merge: [ATT_GROUP][NCW], same, [ATT_GROUP][NCW][64]  (wacc doubles as the cross-attention query scratch)
    float* sqkv;                         // [ATT_GROUP][3][64]: this step's q / k / v of the group's (row, head) tasks
};

// Everything a phase needs, in one place (passed by reference to the __noinline__ phase functions).
struct Env {
    const StepParams* p;
    Smem s;
    int cta, n_cta, pos;
    uint32_t it;          // weight-ring position of the compute side (kept in step by all compute threads)
    uint32_t n_item;      // items this CTA has run (selects the accumulator)
    unsigned nbar;        // grid barriers passed
};

__device__ __forceinline__ Smem carve(unsigned char* sm, const StepParams& p) {
    Smem s;
    s.ring = sm;
    s.act = sm + (size_t)p.n_stage * TILE_BYTES;
    unsigned char* q = s.act + p.act_bytes;
    s.full = reinterpret_cast<uint64_t*>(q);
    s.empty = s.full + MAX_STAGE;
    float* f = reinterpret_cast<float*>(s.empty + MAX_STAGE + 2);
    s.red = f; f += 2 * NCW;
    s.wm = f; f += ATT_GROUP * NCW;
    s.wl = f; f += ATT_GROUP * NCW;
    s.wacc = f; f += ATT_GROUP * NCW * 64;
    s.sqkv = f; f += ATT_GROUP * 192;
    return s;
}

// Which CTA runs item i of GEMM gi in layer `layer`: rotate so that the few SMs without an item differ per GEMM.
__device__ __forceinline__ int cta_rank(int cta, int gi, int layer, int n_cta) {
    return (cta + gi * 53 + layer * 17) % n_cta;
}

__device__ __forceinline__ void stamp(unsigned long long* dst) {
    unsigned long long now;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
    *dst = now;
}

// ------------------------------------------------------------------------------------------------ producer warp
// Walks the step's GEMMs in execution order and keeps the ring full: stage s of use n is handed over on full[s] with
// parity (n & 1) and taken back on empty[s] (one arrival per compute warp once the MMAs reading it have completed).
// A second cursor runs p.l2_ahead tiles further down the same sequence and only issues cp.async.bulk.prefetch.L2: the ring
// covers a fraction of a layer, so without it every GEMM phase re-fills the ring straight from HBM in a burst; with it HBM
// streams at its own pace into L2 and the ring re-fills from L2.
struct TileCursor {
    int g, item, kb, layer, gi;
    const __half* src;      // tile (item, kb)
};
__device__ __forceinline__ void cursor_item(const StepParams& p, TileCursor& c) {
    const StepGemm& G = p.g[c.gi];
    const int nt = c.item / G.ksplit, ks = c.item - nt * G.ksplit;
    c.src = G.wp + (size_t)c.layer * G.layer_stride + ((size_t)nt * G.nkb + (size_t)ks * G.kb_per) * TILE_HALVES;
    c.kb = 0;
}
__device__ __forceinline__ bool cursor_load(const StepParams& p, TileCursor& c, int cta, int n_cta, int total, int per_layer) {
    // position the cursor on GEMM c.g (first item of this CTA); false when the step's GEMMs are exhausted
    for (; c.g < total; ++c.g) {
        c.layer = c.g / per_layer;
        const int k = c.g - c.layer * per_layer;
        c.gi = c.layer == p.L ? SG_HEADS : (p.has_cross ? k : (k < 2 ? k : k + 2));
        if (c.gi == SG_HEADS) c.layer = 0;
        c.item = cta_rank(cta, c.gi, c.layer, n_cta);
        if (c.item < p.g[c.gi].n_items) { cursor_item(p, c); return true; }
    }
    return false;
}
__device__ __forceinline__ const __half* cursor_tile(const StepParams&, const TileCursor& c) { return c.src; }
__device__ __forceinline__ bool cursor_next(const StepParams& p, TileCursor& c, int cta, int n_cta, int total, int per_layer) {
    const StepGemm& G = p.g[c.gi];
    c.src += TILE_HALVES;
    if (++c.kb < G.kb_per) return true;          // the common case: one add and one compare per tile
    c.item += n_cta;
    if (c.item < G.n_items) { cursor_item(p, c); return true; }
    ++c.g;
    return cursor_load(p, c, cta, n_cta, total, per_layer);
}

__device__ __forceinline__ void producer_loop(const StepParams& p, const Smem& s, int cta, int n_cta) {
    const int per_layer = p.has_cross ? 6 : 4;
    int total = p.L * per_layer + 1;
    if (total > p.max_gemms) total = p.max_gemms;   // debug stop (ACB_LM_STEP_STOP): the compute warps leave before the rest
    TileCursor ld{}, pf{};
    bool pf_ok = cursor_load(p, pf, cta, n_cta, total, per_layer);
    for (int i = 0; i < p.l2_ahead && pf_ok; ++i) {   // prime the L2 cursor
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(cursor_tile(p, pf)), "r"((uint32_t)TILE_BYTES) : "memory");
        pf_ok = cursor_next(p, pf, cta, n_cta, total, per_layer);
    }
    uint32_t it = 0;
    if (!cursor_load(p, ld, cta, n_cta, total, per_layer)) return;
#pragma unroll 1
    for (;;) {
        if (pf_ok) {
            asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(cursor_tile(p, pf)), "r"((uint32_t)TILE_BYTES) : "memory");
            pf_ok = cursor_next(p, pf, cta, n_cta, total, per_layer);
        }
        const uint32_t st = it % (uint32_t)p.n_stage, par = (it / (uint32_t)p.n_stage) & 1u;
        mbar_wait_backoff(s.empty + st, par ^ 1u, 200);   // ring full: sleep, do not steal issue slots
        mbar_expect_tx(s.full + st, TILE_BYTES);
        bulk_g2s(s.ring + (size_t)st * TILE_BYTES, cursor_tile(p, ld), TILE_BYTES, s.full + st);
        ++it;
        if (!cursor_next(p, ld, cta, n_cta, total, per_layer)) return;
    }
}

// ------------------------------------------------------------------------------------------------ compute side
// LayerNorm statistics of row r from the per-chunk (mean, M2) records (Chan's merge, equal counts); every thread does
// this for the one row it stages, together with its activation loads, so the GEMM needs no separate statistics pass.
__device__ __forceinline__ void row_mean_rstd(const StepParams& p, int r, float& mean, float& rstd) {
    float2 rec[ACB_STEP_STAT_CHUNKS];
#pragma unroll
    for (int c = 0; c < ACB_STEP_STAT_CHUNKS; ++c)
        rec[c] = __ldcg(reinterpret_cast<const float2*>(p.stats + ((size_t)c * p.R + r) * 2));
    float m = 0.f, m2 = 0.f;
#pragma unroll
    for (int c = 0; c < ACB_STEP_STAT_CHUNKS; ++c) { m += rec[c].x; m2 += rec[c].y; }
    m *= 1.f / ACB_STEP_STAT_CHUNKS;
    float dev = 0.f;
#pragma unroll
    for (int c = 0; c < ACB_STEP_STAT_CHUNKS; ++c) { const float dl = rec[c].x - m; dev = fmaf(dl, dl, dev); }
    m2 += dev * (float)(p.d / ACB_STEP_STAT_CHUNKS);
    mean = m;
    rstd = 1.f / sqrtf(m2 / (float)p.d + 1e-5f);
}

// The MMAs and the epilogue of one GEMM item: warpgroup g multiplies features [64 g, +64) of the ring's weight tiles with the
// staged [R][64] activation tiles.  The K steps rotate over NACC independent accumulators that the epilogue adds in a fixed
// order, so every partial sum is the same whatever the pipelining of the MMAs.  Every compute warp arrives on the empty
// barrier of a stage once its warpgroup's MMAs on it have completed.  At R = 64 the NACC accumulators take 128 registers per
// thread and ptxas reports spills in lm_step_kernel; their cost on the H100 has not been measured.
template <int R>
__device__ __forceinline__ void gemm_item_mma(Env& e, const StepGemm& G, int layer, int gi, int nt, int ks, bool trc) {
    const StepParams& p = *e.p;
    const Smem& s = e.s;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = __shfl_sync(0xffffffffu, warp >> 2, 0);   // warpgroup, provably warp-uniform
    const uint32_t act_s = smem_u32(s.act), ring_s = smem_u32(s.ring) + (uint32_t)g * (64u * 128u);
    float acc[NACC][R / 2];
#pragma unroll
    for (int a = 0; a < NACC; ++a)
#pragma unroll
        for (int i = 0; i < R / 2; ++i) acc[a][i] = 0.f;
    uint32_t it = e.it;
#pragma unroll 1
    for (int kb = 0; kb < G.kb_per; ++kb, ++it) {
        const uint32_t st = it % (uint32_t)p.n_stage, par = (it / (uint32_t)p.n_stage) & 1u;
        const bool trk = trc && tid == 0 && layer == 1 && (gi == SG_FF2 || gi == SG_QKV);   // per-K-block stamps of two GEMMs of layer 1
        if (trk) stamp(p.trace + 6000 + (gi == SG_FF2 ? 64 : 0) + 3 * kb);
        mbar_wait(s.full + st, par);
        if (trk) stamp(p.trace + 6000 + (gi == SG_FF2 ? 64 : 0) + 3 * kb + 1);
        const uint32_t a_s = ring_s + st * (uint32_t)TILE_BYTES, b_s = act_s + (uint32_t)kb * (uint32_t)R * 128u;
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) {   // one instruction = 16 K elements = 32 bytes along the swizzled row
            wgmma_fence_regs(acc[j % NACC]);
            wgmma_f16<R>(acc[j % NACC], wgmma_desc_sw128(a_s + 32u * j), wgmma_desc_sw128(b_s + 32u * j), kb * 4 + j >= NACC ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int a = 0; a < NACC; ++a) wgmma_fence_regs(acc[a]);
        __syncwarp();
        if (lane == 0) mbar_arrive(s.empty + st);   // stage free again once both warpgroups have read it
        if (trk) stamp(p.trace + 6000 + (gi == SG_FF2 ? 64 : 0) + 3 * kb + 2);
    }
    // thread (warp w of the warpgroup, lane l): features 64 g + 16 w + l / 4 (+ 8), rows 8 j + 2 (l % 4) (+ 1)
    float* out = p.part + ((size_t)ks * R) * G.N + (size_t)nt * 128 + g * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int i = 0; i < R / 2; ++i) {
        float sum = acc[0][i];
#pragma unroll
        for (int a = 1; a < NACC; ++a) sum += acc[a][i];   // fixed order
        const int r = (i >> 2) * 8 + (lane & 3) * 2 + (i & 1);
        if (r < p.rows) out[(size_t)r * G.N + ((i >> 1) & 1) * 8] = sum;
    }
}

// One GEMM of the step.  gamma != NULL: the activations are LayerNorm(x) (statistics from the residual phase, gamma / beta
// applied in fp32, rounded to fp16 like the reference's autocast LayerNorm -> Linear); else they are the fp16 rows of src16.
__device__ __forceinline__ void gemm_phase(Env& e, int gi, int layer, const float* gamma, const float* beta, const __half* src16, int ld16) {
    const StepParams& p = *e.p;
    const Smem& s = e.s;
    const StepGemm& G = p.g[gi];
    const int tid = threadIdx.x;
    const int R = p.R, rows = p.rows;
    const int first = cta_rank(e.cta, gi, layer, e.n_cta);
    if (first >= G.n_items) return;
    const bool trc = p.trace != nullptr && first == 0;   // this CTA traces its sub-steps
    const bool tr = trc && tid == 0;
    if (tr) stamp(p.trace + 1024 + 8 * e.nbar);
#pragma unroll 1
    for (int item = first; item < G.n_items; item += e.n_cta) {
        const int nt = item / G.ksplit, ks = item - nt * G.ksplit;
        const int k0 = ks * G.kb_per * 64, nch2 = G.kb_per * 4;
        // ---- stage the activations [rows][k0 .. k0 + 64*kb_per) as the B operand, one [R][64] tile per K block
        //      (stored in the 128-byte-swizzled K-major operand layout, see wgmma_desc_sw128)
        //      A thread stages (row, two 16-byte chunks) per iteration; with 512 threads that is one iteration for the
        //      medium model, and all of an iteration's loads (statistics included) are independent.
#pragma unroll 1
        for (int idx = tid; idx < rows * nch2; idx += CT) {
            const int c2 = idx / rows, r = idx - c2 * rows;
            const int k = k0 + c2 * 16;
            uint4 o0, o1;
            if (gamma) {
                const float* xr = p.x + (size_t)r * p.d + k;
                const float4 a0 = ldcg4(xr), a1 = ldcg4(xr + 4), a2 = ldcg4(xr + 8), a3 = ldcg4(xr + 12);
                float mu, rs;
                row_mean_rstd(p, r, mu, rs);
                const float4* gp = reinterpret_cast<const float4*>(gamma + k);
                const float4* bp = reinterpret_cast<const float4*>(beta + k);
                float4 g = __ldg(gp), b = __ldg(bp);
                o0.x = pack_h2((a0.x - mu) * rs * g.x + b.x, (a0.y - mu) * rs * g.y + b.y);
                o0.y = pack_h2((a0.z - mu) * rs * g.z + b.z, (a0.w - mu) * rs * g.w + b.w);
                g = __ldg(gp + 1); b = __ldg(bp + 1);
                o0.z = pack_h2((a1.x - mu) * rs * g.x + b.x, (a1.y - mu) * rs * g.y + b.y);
                o0.w = pack_h2((a1.z - mu) * rs * g.z + b.z, (a1.w - mu) * rs * g.w + b.w);
                g = __ldg(gp + 2); b = __ldg(bp + 2);
                o1.x = pack_h2((a2.x - mu) * rs * g.x + b.x, (a2.y - mu) * rs * g.y + b.y);
                o1.y = pack_h2((a2.z - mu) * rs * g.z + b.z, (a2.w - mu) * rs * g.w + b.w);
                g = __ldg(gp + 3); b = __ldg(bp + 3);
                o1.z = pack_h2((a3.x - mu) * rs * g.x + b.x, (a3.y - mu) * rs * g.y + b.y);
                o1.w = pack_h2((a3.z - mu) * rs * g.z + b.z, (a3.w - mu) * rs * g.w + b.w);
            } else {
                const uint4* sp = reinterpret_cast<const uint4*>(src16 + (size_t)r * ld16 + k);
                o0 = __ldcg(sp);
                o1 = __ldcg(sp + 1);
            }
            // K block kb = c2 / 4 holds this row's 128 bytes at kb * R * 128 + r * 128; chunk c goes to position c ^ (r & 7)
            unsigned char* dst = s.act + ((size_t)(c2 >> 2) * R + r) * 128;
            const int c = (c2 & 3) * 2, sw = r & 7;
            *reinterpret_cast<uint4*>(dst + ((c ^ sw) << 4)) = o0;
            *reinterpret_cast<uint4*>(dst + (((c + 1) ^ sw) << 4)) = o1;
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
        cbar();
        if (tr) stamp(p.trace + 1024 + 8 * e.nbar + 2);
        switch (R) {
            case 16: gemm_item_mma<16>(e, G, layer, gi, nt, ks, trc); break;
            case 32: gemm_item_mma<32>(e, G, layer, gi, nt, ks, trc); break;
            case 48: gemm_item_mma<48>(e, G, layer, gi, nt, ks, trc); break;
            default: gemm_item_mma<64>(e, G, layer, gi, nt, ks, trc); break;
        }
        e.it += (uint32_t)G.kb_per;
        ++e.n_item;
        cbar();   // activation tile reusable
        if (tr) stamp(p.trace + 1024 + 8 * e.nbar + 5);
    }
}

// sum over the CT compute threads; `red` holds NCW floats and is reusable after the NEXT cbar()
__device__ __forceinline__ float cw_sum(float v, float* red) {
    v = warp_sum(v);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) red[warp] = v;
    cbar();
    float t = lane < NCW ? red[lane] : 0.f;
    return warp_sum(t);
}

// x[r][col] for the embed phase: sum_k emb_k[token] + sinusoidal position (lm.py:244, transformer.py:70-89, 701-705).
// Runs once per step: kept out of residual_phase so that its sin / cos code is not part of the per-layer footprint.
__device__ __noinline__ float embed_value(const StepParams& p, int r, int col, int pos) {
    const int d = p.d, b = r % p.batch, half_d = d >> 1;
    float v = 0.f;
#pragma unroll 1
    for (int k = 0; k < p.n_q; ++k) {
        long long tk = p.seq[((size_t)b * p.n_q + k) * p.max_seq + pos];
        const int tok = (int)(tk < 0 ? p.card : (tk > p.card ? p.card : tk));
        v += __half2float(p.emb[((size_t)k * (p.card + 1) + tok) * d + col]);
    }
    if (p.sin_pos) {
        const int j = col < half_d ? col : col - half_d;
        const float phase = (float)pos / p.inv_freq[j];
        v += p.pos_scale * (col < half_d ? cosf(phase) : sinf(phase));
    }
    return v;
}

// x[r][cols of chunk c] += sum of the split-K partials (fixed order), and the chunk's LayerNorm record (mean, centred sum
// of squares).  embed != 0: x = the step's input embedding instead.
__device__ __forceinline__ void residual_phase(Env& e, int ksplit, int embed) {
    const StepParams& p = *e.p;
    const int tid = threadIdx.x, d = p.d, len = d / ACB_STEP_STAT_CHUNKS, tasks = p.rows * ACB_STEP_STAT_CHUNKS;
#pragma unroll 1
    for (int t = e.cta; t < tasks; t += e.n_cta) {
        const int c = t / p.rows, r = t - c * p.rows;
        const bool live = tid < len;
        const int col = c * len + tid;
        float v = 0.f;
        if (live) {
            if (embed) {
                v = embed_value(p, r, col, e.pos);
            } else {
                const float* pp = p.part + (size_t)r * d + col;
                const size_t stride = (size_t)p.R * d;
                v = __ldcg(p.x + (size_t)r * d + col);
#pragma unroll 1
                for (int k0 = 0; k0 < ksplit; k0 += 8) {   // 8 independent loads in flight, summed in slot order
                    float pv[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) pv[j] = k0 + j < ksplit ? __ldcg(pp + (size_t)(k0 + j) * stride) : 0.f;
#pragma unroll
                    for (int j = 0; j < 8; ++j) v += pv[j];
                }
            }
            p.x[(size_t)r * d + col] = v;
        }
        const float mean = cw_sum(live ? v : 0.f, e.s.red) / (float)len;
        const float dv = live ? v - mean : 0.f;
        const float m2 = cw_sum(dv * dv, e.s.red + NCW);
        if (tid == 0) *reinterpret_cast<float2*>(p.stats + ((size_t)c * p.R + r) * 2) = make_float2(mean, m2);
        cbar();
    }
}

// mode 0: h16[r][n] = gelu(fp16(sum of the FF1 partials))  (linear1's output is fp16 under autocast, then F.gelu, transformer.py:569)
// mode 1: logits[r][n] = sum of the heads' partials
__device__ __forceinline__ void sum_phase(Env& e, int ksplit, int N, int mode) {
    const StepParams& p = *e.p;
    const int n4 = N >> 2, total = p.rows * n4;
    const size_t stride = (size_t)p.R * N;
#pragma unroll 1
    for (int g = e.cta * CT + threadIdx.x; g < total; g += e.n_cta * CT) {
        const int r = g / n4, c4 = g - r * n4;
        const float* pp = p.part + (size_t)r * N + c4 * 4;
        float a[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
        for (int k0 = 0; k0 < ksplit; k0 += 4) {
            float4 pv[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) pv[j] = k0 + j < ksplit ? ldcg4(pp + (size_t)(k0 + j) * stride) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int j = 0; j < 4; ++j) { a[0] += pv[j].x; a[1] += pv[j].y; a[2] += pv[j].z; a[3] += pv[j].w; }
        }
        if (mode == 0) {
#pragma unroll 1
            for (int j = 0; j < 4; ++j) {   // rolled: ONE copy of erff
                const float h = half_round(a[j]);
                a[j] = 0.5f * h * (1.f + erff(h * 0.70710678118654752440f));
            }
            uint2 pk;
            pk.x = pack_h2(a[0], a[1]); pk.y = pack_h2(a[2], a[3]);
            *reinterpret_cast<uint2*>(p.h16 + (size_t)r * N + c4 * 4) = pk;
        } else {
            *reinterpret_cast<float4*>(p.logits + (size_t)r * N + c4 * 4) = make_float4(a[0], a[1], a[2], a[3]);
        }
    }
}

struct OnlineSM { float m, l, acc[8]; };
__device__ __forceinline__ void osm_merge(OnlineSM& a, float m2, float l2, const float (&acc2)[8]) {
    const float mn = fmaxf(a.m, m2);
    const float ca = a.m == -INFINITY ? 0.f : __expf(a.m - mn), cb = m2 == -INFINITY ? 0.f : __expf(m2 - mn);
    a.l = a.l * ca + l2 * cb;
#pragma unroll
    for (int e = 0; e < 8; ++e) a.acc[e] = a.acc[e] * ca + acc2[e] * cb;
    a.m = mn;
}
__device__ __forceinline__ void osm_step(OnlineSM& st, float sc, const uint4& vraw) {
    const float mn = fmaxf(st.m, sc);
    const float corr = __expf(st.m - mn);   // exp(-inf) = 0 on the first position
    const float pw = __expf(sc - mn);
    st.l = st.l * corr + pw;
    const __half2* v2 = reinterpret_cast<const __half2*>(&vraw);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(v2[e]);
        st.acc[2 * e] = fmaf(pw, f.x, st.acc[2 * e] * corr);
        st.acc[2 * e + 1] = fmaf(pw, f.y, st.acc[2 * e + 1] * corr);
    }
    st.m = mn;
}
// q . k over the 8 dims this lane holds, reduced over the 8 lanes of a position
__device__ __forceinline__ float qk_dot(const float (&q)[8], const uint4& kraw) {
    const __half2* k2 = reinterpret_cast<const __half2*>(&kraw);
    float sc = 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(k2[e]);
        sc = fmaf(q[2 * e], f.x, sc);
        sc = fmaf(q[2 * e + 1], f.y, sc);
    }
    sc += __shfl_xor_sync(0xffffffffu, sc, 1);
    sc += __shfl_xor_sync(0xffffffffu, sc, 2);
    sc += __shfl_xor_sync(0xffffffffu, sc, 4);
    return sc;
}

// RotaryEmbedding.rotate_qk (modules/rope.py:84-125) on one fp16 element of q / k at position pos: the head dim is 32 complex
// pairs (2i, 2i+1), rotated by pos * max_period^(-2i/64) in fp32 and blended with `scale`; `other` is the pair partner.
// Out of line: sincosf is large and rotary positions are an option, not the released models' default.
__device__ __noinline__ float rope_rotate(const StepParams& p, float vh, float other, int dd, int pos) {
    const bool even = (dd & 1) == 0;
    const float re = even ? vh : other, im = even ? other : vh;
    const float ang = (float)pos * p.rope_freq[dd >> 1];
    float sn, cs;
    sincosf(ang, &sn, &cs);
    const float rr = cs * p.pos_scale + (1.f - p.pos_scale), ri = sn * p.pos_scale;
    return even ? re * rr - im * ri : re * ri + im * rr;
}

// Self-attention of the step's single query per (row, head): sums the QKV partials of the head, applies the rotary
// embedding when configured, appends k / v to the cache (fp16, like the reference's cached fp16 keys), then one
// online-softmax pass over the cache (StreamingMultiheadAttention.forward, transformer.py:315-451, cache :266-298).
__device__ __forceinline__ void self_attn_phase(Env& e, int layer) {
    const StepParams& p = *e.p;
    const Smem& s = e.s;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, sl = lane & 7, pg = lane >> 3;
    const int d = p.d, H = p.H, R = p.R, N3 = 3 * d, ksplit = p.g[SG_QKV].ksplit, pos = e.pos;
    const size_t kv_layer = (size_t)p.max_rows * H * p.max_seq * 64;
    __half* kc = p.kc + (size_t)layer * kv_layer;
    __half* vc = p.vc + (size_t)layer * kv_layer;
    const int tasks = p.rows * H;
    const int t_first = (e.cta + layer * 29) % e.n_cta;
    // A CTA's tasks t_first, t_first + n_cta, ... are handled ATT_GROUP at a time: one pass sums the QKV partials of the whole
    // group (all loads in flight together), one barrier, the KV streams task by task, one barrier, one merge pass.
#pragma unroll 1
    for (int t0 = t_first; t0 < tasks; t0 += ATT_GROUP * e.n_cta) {
        const int n_here = min(ATT_GROUP, (tasks - t0 + e.n_cta - 1) / e.n_cta);
        // ---- stage 1: q / k / v of this step for every task of the group (fixed-order partial sums; k, v appended to the cache)
#pragma unroll 1
        for (int el = tid; el < n_here * 192; el += CT) {
            const int j = el / 192, rem = el - j * 192, which = rem >> 6, dd = rem & 63;
            const int t = t0 + j * e.n_cta, row = t / H, h = t - row * H;
            const float* src = p.part + (size_t)row * N3 + which * d + h * 64 + dd;
            const size_t stride = (size_t)R * N3;
            float v = 0.f;
#pragma unroll 1
            for (int k0 = 0; k0 < ksplit; k0 += 4) {   // 4 independent loads in flight, summed in slot order
                float pv[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) pv[i] = k0 + i < ksplit ? __ldcg(src + (size_t)(k0 + i) * stride) : 0.f;
#pragma unroll
                for (int i = 0; i < 4; ++i) v += pv[i];
            }
            if (p.rope && which < 2) {   // (192 = 6 warps per task: a warp holds 32 consecutive dims of one of q / k / v)
                const float vh = half_round(v);
                v = rope_rotate(p, vh, __shfl_xor_sync(0xffffffffu, vh, 1), dd, pos);
            }
            if (which == 0) {
                s.sqkv[j * 192 + dd] = half_round(v) * p.attn_scale;
            } else {
                const __half hv = __float2half_rn(v);
                (which == 1 ? kc : vc)[(((size_t)row * H + h) * p.max_seq + pos) * 64 + dd] = hv;
                s.sqkv[j * 192 + which * 64 + dd] = __half2float(hv);
            }
        }
        cbar();
        // ---- stage 2: one online-softmax pass over each task's cache, positions split over the warps
#pragma unroll 1
        for (int j = 0; j < n_here; ++j) {
            const int t = t0 + j * e.n_cta, row = t / H, h = t - row * H;
            const size_t base = ((size_t)row * H + h) * p.max_seq * 64;
            const float* sq = s.sqkv + j * 192;
            float q[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) q[i] = sq[sl * 8 + i];
            OnlineSM st;
            st.m = -INFINITY; st.l = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) st.acc[i] = 0.f;
            const __half* kb = kc + base + sl * 8;
            const __half* vb = vc + base + sl * 8;
            // cached positions [0, pos): a warp instruction reads 4 consecutive positions (512 contiguous bytes); a lane keeps
            // the K / V vectors of the batch being consumed AND of the next batch in registers (software pipeline): with one
            // CTA per SM nothing else hides the HBM latency of this stream.
            {
                constexpr int STRIDE = NCW * 4 * ATT_UNROLL;
                uint4 ka[ATT_UNROLL], va[ATT_UNROLL], kn[ATT_UNROLL], vn[ATT_UNROLL];
                int pb = warp * 4;                       // warp-uniform loop bounds (the shuffles need all 32 lanes)
                if (pb < pos) {
#pragma unroll
                    for (int u = 0; u < ATT_UNROLL; ++u) {
                        const int pp = pb + u * NCW * 4 + pg;
                        ka[u] = pp < pos ? ld_stream_u4(kb + (size_t)pp * 64) : make_uint4(0, 0, 0, 0);
                        va[u] = pp < pos ? ld_stream_u4(vb + (size_t)pp * 64) : make_uint4(0, 0, 0, 0);
                    }
                }
#pragma unroll 1
                while (pb < pos) {
                    const int nb = pb + STRIDE;
                    if (nb < pos) {
#pragma unroll
                        for (int u = 0; u < ATT_UNROLL; ++u) {
                            const int pp = nb + u * NCW * 4 + pg;
                            kn[u] = pp < pos ? ld_stream_u4(kb + (size_t)pp * 64) : make_uint4(0, 0, 0, 0);
                            vn[u] = pp < pos ? ld_stream_u4(vb + (size_t)pp * 64) : make_uint4(0, 0, 0, 0);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < ATT_UNROLL; ++u) {
                        const float sc = qk_dot(q, ka[u]);
                        if (pb + u * NCW * 4 + pg < pos) osm_step(st, sc, va[u]);
                    }
#pragma unroll
                    for (int u = 0; u < ATT_UNROLL; ++u) { ka[u] = kn[u]; va[u] = vn[u]; }
                    pb = nb;
                }
            }
            if (warp == 0) {   // the position appended by this step, from shared memory
                float sc = 0.f;
#pragma unroll
                for (int i = 0; i < 8; ++i) sc = fmaf(q[i], sq[64 + sl * 8 + i], sc);
                sc += __shfl_xor_sync(0xffffffffu, sc, 1);
                sc += __shfl_xor_sync(0xffffffffu, sc, 2);
                sc += __shfl_xor_sync(0xffffffffu, sc, 4);
                if (pg == 0) {
                    const float mn = fmaxf(st.m, sc), corr = __expf(st.m - mn), pw = __expf(sc - mn);
                    st.l = st.l * corr + pw;
#pragma unroll
                    for (int i = 0; i < 8; ++i) st.acc[i] = fmaf(pw, sq[128 + sl * 8 + i], st.acc[i] * corr);
                    st.m = mn;
                }
            }
            // merge the 4 position groups of the warp; the warps are merged in stage 3
#pragma unroll
            for (int o = 8; o <= 16; o <<= 1) {
                const float m2 = __shfl_xor_sync(0xffffffffu, st.m, o), l2 = __shfl_xor_sync(0xffffffffu, st.l, o);
                float a2[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) a2[i] = __shfl_xor_sync(0xffffffffu, st.acc[i], o);
                osm_merge(st, m2, l2, a2);
            }
            if (pg == 0) {
                if (sl == 0) { s.wm[j * NCW + warp] = st.m; s.wl[j * NCW + warp] = st.l; }
#pragma unroll
                for (int i = 0; i < 8; ++i) s.wacc[(j * NCW + warp) * 64 + sl * 8 + i] = st.acc[i];
            }
        }
        cbar();
        // ---- stage 3: merge the warps' partial softmaxes, one thread per output dim of every task of the group
        if (tid < n_here * 64) {
            const int j = tid >> 6, dd = tid & 63;
            const int t = t0 + j * e.n_cta, row = t / H, h = t - row * H;
            const float* wm = s.wm + j * NCW;
            float mx = -INFINITY;
#pragma unroll
            for (int w = 0; w < NCW; ++w) mx = fmaxf(mx, wm[w]);
            float l = 0.f, o = 0.f;
#pragma unroll
            for (int w = 0; w < NCW; ++w) {
                const float cw = wm[w] == -INFINITY ? 0.f : __expf(wm[w] - mx);
                l = fmaf(s.wl[j * NCW + w], cw, l);
                o = fmaf(s.wacc[(j * NCW + w) * 64 + dd], cw, o);
            }
            p.a16[(size_t)row * d + h * 64 + dd] = __float2half_rn(o / l);
        }
        cbar();   // scratch reusable by the next group
    }
}

// Cross-attention over the cached text keys / values (computed once per generate): one warp per (row, head); the padded
// / null text positions are zero keys that still take part in the softmax (conditioners.py:1731-1746, transformer.py:343).
__device__ __forceinline__ void cross_attn_phase(Env& e, int layer) {
    const StepParams& p = *e.p;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int d = p.d, H = p.H, R = p.R, ksplit = p.g[SG_CQ].ksplit, n = p.text_len;
    const size_t ckv_layer = (size_t)p.max_rows * H * p.max_text * 64;
    const __half* kc = p.ckc + (size_t)layer * ckv_layer;
    const __half* vc = p.cvc + (size_t)layer * ckv_layer;
    float* qs = e.s.wacc + warp * 64;
    const int tasks = p.rows * H;
#pragma unroll 1
    for (int t = (e.cta + layer * 31) % e.n_cta + e.n_cta * warp; t < tasks; t += e.n_cta * NCW) {
        const int row = t / H, h = t - row * H;
        {
            const float* qp = p.part + (size_t)row * d + h * 64 + lane * 2;
            const size_t stride = (size_t)R * d;
            float a0 = 0.f, a1 = 0.f;
#pragma unroll 1
            for (int k0 = 0; k0 < ksplit; k0 += 8) {   // 8 independent loads in flight, summed in slot order
                float2 pv[8];
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    pv[j] = k0 + j < ksplit ? __ldcg(reinterpret_cast<const float2*>(qp + (size_t)(k0 + j) * stride)) : make_float2(0.f, 0.f);
#pragma unroll
                for (int j = 0; j < 8; ++j) { a0 += pv[j].x; a1 += pv[j].y; }
            }
            qs[lane * 2] = half_round(a0) * p.attn_scale;
            qs[lane * 2 + 1] = half_round(a1) * p.attn_scale;
        }
        __syncwarp();
        const size_t base = ((size_t)row * H + h) * p.max_text * 64;
        float mx = -INFINITY, l = 0.f, o0 = 0.f, o1 = 0.f;
#pragma unroll 1
        for (int t0 = 0; t0 < n; t0 += 32) {
            const int tt = t0 + lane;
            float sc = -INFINITY;
            if (tt < n) {
                const uint4* kr = reinterpret_cast<const uint4*>(kc + base + (size_t)tt * 64);
                uint4 kk[8];
#pragma unroll
                for (int c8 = 0; c8 < 8; ++c8) kk[c8] = kr[c8];
                sc = 0.f;
#pragma unroll
                for (int c8 = 0; c8 < 8; ++c8) {
                    const __half2* k2 = reinterpret_cast<const __half2*>(&kk[c8]);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float2 f = __half22float2(k2[i]);
                        sc = fmaf(qs[c8 * 8 + 2 * i], f.x, sc);
                        sc = fmaf(qs[c8 * 8 + 2 * i + 1], f.y, sc);
                    }
                }
            }
            const float cm = fmaxf(mx, warp_max(sc));
            const float corr = mx == -INFINITY ? 0.f : __expf(mx - cm);
            const float pw = tt < n ? __expf(sc - cm) : 0.f;
            l = l * corr + warp_sum(pw);
            o0 *= corr; o1 *= corr;
            const int cnt = min(32, n - t0);
            const __half* vp = vc + base + (size_t)t0 * 64 + lane * 2;
#pragma unroll 1
            for (int j0 = 0; j0 < cnt; j0 += 8) {   // 8 value rows in flight
                __half2 vv[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) vv[j] = j0 + j < cnt ? *reinterpret_cast<const __half2*>(vp + (size_t)(j0 + j) * 64) : __half2();
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float wj = __shfl_sync(0xffffffffu, pw, (j0 + j) & 31);
                    const float2 f = __half22float2(vv[j]);
                    if (j0 + j < cnt) { o0 = fmaf(wj, f.x, o0); o1 = fmaf(wj, f.y, o1); }
                }
            }
            mx = cm;
        }
        *reinterpret_cast<__half2*>(p.a16 + (size_t)row * d + h * 64 + lane * 2) = __floats2half2_rn(o0 / l, o1 / l);
        __syncwarp();
    }
}

// grid barrier at the end of a phase; true = the debug stop point (p.stop_after barriers) has been reached
__device__ __forceinline__ bool phase_end(Env& e) {
    const StepParams& p = *e.p;
    cbar();
    ++e.nbar;
    if (threadIdx.x == ISSUE_WARP * 32) {
        gridbar_arrive(p.bar);
        gridbar_wait(p.bar, e.nbar * (unsigned)e.n_cta);   // the other warps are blocked in bar.sync: nothing to starve
        if (p.trace && e.cta == 0) stamp(p.trace + e.nbar);
    }
    cbar();
    return (int)e.nbar >= p.stop_after;
}

// The compute warps' program: ONE loop over the step's phases with each phase kind's code appearing exactly once (inlined:
// kernel parameters come from the constant bank and the running state stays in registers -- behind __noinline__ calls both
// sat in memory that the gpu-scope acquire of every grid barrier invalidates in L1, costing each phase several L2 round trips
// before it had loaded a single operand).  Phase p > 0 of layer l = (p - 1) / per, kind k = (p - 1) % per:
//   0 QKV gemm | 1 self-attention | 2 O gemm | 3 residual | 4 CQ gemm | 5 cross-attention | 6 CO gemm | 7 residual |
//   8 FF1 gemm | 9 gelu | 10 FF2 gemm | 11 residual        (k = 4..7 absent without cross attention)
// then the heads gemm and the logits sum.  GEMM k runs step GEMM k / 2 (the SG_* order).
__device__ __forceinline__ void consumer_body(Env& e) {
    const StepParams& p = *e.p;
    const int d = p.d, per = p.has_cross ? 12 : 8, n_layer_ph = p.L * per, n_ph = 1 + n_layer_ph + 2;
#pragma unroll 1
    for (int ph = 0; ph < n_ph; ++ph) {
        int kind, layer = 0, k = 0;            // kind: 0 gemm, 1 self-attn, 2 cross-attn, 3 residual, 4 sum, 5 embed
        if (ph == 0) {
            kind = 5;
        } else if (ph <= n_layer_ph) {
            layer = (ph - 1) / per;
            k = (ph - 1) - layer * per;
            if (!p.has_cross && k >= 4) k += 4;
            kind = (k & 1) == 0 ? 0 : (k == 1 ? 1 : (k == 5 ? 2 : (k == 9 ? 4 : 3)));
        } else {
            kind = ph == n_layer_ph + 1 ? 0 : 4;
            k = 12;                            // heads
        }
        if (kind == 0) {
            const int gi = k >> 1;             // 0..5 in a layer, 6 = heads
            const float* ln = gi == SG_HEADS ? p.out_norm : p.ln + (size_t)layer * 6 * d + (size_t)gi * d;   // k/2 = 0, 2, 4 -> norm1, norm_cross, norm2
            const bool is_ln = gi == SG_QKV || gi == SG_CQ || gi == SG_FF1 || gi == SG_HEADS;
            const __half* src = gi == SG_FF2 ? p.h16 : p.a16;
            gemm_phase(e, gi, layer, is_ln ? ln : nullptr, is_ln ? ln + d : nullptr, src, gi == SG_FF2 ? p.ffn : d);
            if (gi == SG_QKV && layer + 1 < p.L && e.cta == (layer * 7) % e.n_cta) {
                // next layer's LayerNorm parameters (6 d floats) -> L2 now: their first use is otherwise an HBM-latency miss
                const char* nx = reinterpret_cast<const char*>(p.ln + (size_t)(layer + 1) * 6 * d);
                for (int i = threadIdx.x * 128; i < 6 * d * 4; i += CT * 128)
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(nx + i));
            }
        } else if (kind == 1) {
            self_attn_phase(e, layer);
        } else if (kind == 2) {
            cross_attn_phase(e, layer);
        } else if (kind == 3) {
            residual_phase(e, p.g[(k - 1) >> 1].ksplit, 0);
        } else if (kind == 4) {
            if (k == 12) sum_phase(e, p.g[SG_HEADS].ksplit, p.n_q * p.card, 1);
            else sum_phase(e, p.g[SG_FF1].ksplit, p.ffn, 0);
        } else {
            residual_phase(e, 0, 1);
        }
        if (ph + 1 < n_ph && phase_end(e)) return;
    }
}

__global__ void __launch_bounds__(BLOCK, 1) lm_step_kernel(const __grid_constant__ StepParams p) {
    extern __shared__ __align__(1024) unsigned char step_sm[];
    const Smem s = carve(step_sm, p);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int cta = blockIdx.x, n_cta = gridDim.x;

    if (tid == 0) {
        for (int i = 0; i < p.n_stage; ++i) { mbar_init(s.full + i, 1); mbar_init(s.empty + i, NCW); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        if (p.trace && cta == 0) stamp(p.trace);
    }
    for (int i = tid; i < p.act_bytes / 16; i += BLOCK) reinterpret_cast<uint4*>(s.act)[i] = make_uint4(0, 0, 0, 0);   // padded rows stay 0
    __syncthreads();

    if (warp == NCW) {
        if (lane == 0) producer_loop(p, s, cta, n_cta);
    } else {
        Env e;
        e.p = &p; e.s = s; e.cta = cta; e.n_cta = n_cta; e.pos = p.pos[0];
        e.it = 0; e.n_item = 0; e.nbar = 0;
        consumer_body(e);
    }
}

// [N][K] row-major fp16 -> tiles of 128 features x 64 K in the 128-byte-swizzled K-major layout (see wgmma_desc_sw128):
//   tile (nt, kb) at ((nt * nkb + kb) * 8192) halves; inside: row f at f * 128 bytes, its 16-byte chunk c at position c ^ (f & 7)
__global__ void lm_pack_kernel(const __half* __restrict__ src, __half* __restrict__ dst, int N, int K) {
    const int nkb = K >> 6;
    const size_t total = (size_t)N * K / 8;   // 16-byte chunks
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int cpos = (int)(i & 7), f = (int)((i >> 3) & 127);
        const size_t tile = i >> 10;
        const int kb = (int)(tile % nkb), nt = (int)(tile / nkb);
        const int c = cpos ^ (f & 7);
        const uint4 v = *reinterpret_cast<const uint4*>(src + ((size_t)nt * 128 + f) * K + (size_t)kb * 64 + c * 8);
        reinterpret_cast<uint4*>(dst)[i] = v;
    }
}

}  // namespace

extern "C" int acb_lm_pack_weight(const void* w, void* wp, int n, int k, void* stream) {
    ACB_REQUIRE(w && wp && n > 0 && k > 0 && n % 128 == 0 && k % 64 == 0, "acb_lm_pack_weight: N %% 128 and K %% 64 must be 0 (N=%d K=%d)", n, k);
    const size_t total = (size_t)n * k / 8;
    const int blocks = (int)((total + 255) / 256 < 65535 * 16 ? (total + 255) / 256 : 65535 * 16);
    lm_pack_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const __half*)w, (__half*)wp, n, k);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

// K-slices per GEMM: minimise (k-blocks the busiest CTA multiplies) + a charge per split (partial traffic, reduction).
static void plan_gemm(StepGemm& G, const void* wp, size_t layer_stride, int N, int K, int sms, int R) {
    G.wp = (const __half*)wp; G.layer_stride = layer_stride; G.N = N; G.K = K;
    G.n_tiles = N / 128; G.nkb = K / 64;
    float best = 1e30f;
    int best_ks = 1;
    for (int ks = 1; ks <= ACB_STEP_MAX_SPLIT && ks <= G.nkb; ++ks) {
        if (G.nkb % ks) continue;
        const int per = G.nkb / ks;
        if ((size_t)per * 64 * R * 2 > 96 * 1024 || per > 8) continue;   // activation tile (<= 8 K blocks) must fit beside the ring
        const int items = G.n_tiles * ks;
        const float cost = (float)((items + sms - 1) / sms) * per + 0.35f * ks;
        if (cost < best) { best = cost; best_ks = ks; }
    }
    G.ksplit = best_ks; G.kb_per = G.nkb / best_ks; G.n_items = G.n_tiles * best_ks;
}

int lm_step_prepare(const acb_lm_config& c, const acb_lm_weights& w, const acb_lm_buffers& b, int rows, int batch, int text_len,
                    bool has_cross, int sms, StepLaunch* out) {
    const int d = c.dim, ffn = c.ffn_dim, NH = c.n_q * c.card;
    ACB_REQUIRE(w.wp_qkv && w.wp_o && w.wp_ff1 && w.wp_ff2 && w.wp_heads && (!c.cross_attention || (w.wp_cq && w.wp_co)),
                "fused step: packed weights missing");
    ACB_REQUIRE(b.stats && b.part && b.bar, "fused step: stats / part / bar buffers missing");
    ACB_REQUIRE(d % 128 == 0 && ffn % 128 == 0 && NH % 128 == 0, "fused step: dim, ffn and n_q*card must be multiples of 128");
    ACB_REQUIRE(d / ACB_STEP_STAT_CHUNKS <= CT && (d / ACB_STEP_STAT_CHUNKS) >= 1 && d % (8 * ACB_STEP_STAT_CHUNKS) == 0, "fused step: dim %d not supported", d);
    ACB_REQUIRE(rows >= 1 && rows <= 64, "fused step: rows %d not in [1,64]", rows);
    StepLaunch L{};
    StepParams& p = L.p;
    p.d = d; p.H = c.num_heads; p.L = c.num_layers; p.ffn = ffn; p.n_q = c.n_q; p.card = c.card;
    p.rows = rows; p.R = (rows + 15) / 16 * 16; p.batch = batch; p.has_cross = has_cross ? 1 : 0; p.text_len = text_len;
    p.max_seq = c.max_seq; p.max_text = c.max_text; p.max_rows = c.max_rows;
    p.pos_scale = c.pos_scale; p.attn_scale = 1.0f / sqrtf(64.f);
    p.emb = (const __half*)w.emb; p.inv_freq = w.inv_freq; p.ln = w.ln; p.out_norm = w.out_norm;
    plan_gemm(p.g[SG_QKV], w.wp_qkv, (size_t)3 * d * d, 3 * d, d, sms, p.R);
    plan_gemm(p.g[SG_O], w.wp_o, (size_t)d * d, d, d, sms, p.R);
    plan_gemm(p.g[SG_CQ], w.wp_cq, (size_t)d * d, d, d, sms, p.R);
    plan_gemm(p.g[SG_CO], w.wp_co, (size_t)d * d, d, d, sms, p.R);
    plan_gemm(p.g[SG_FF1], w.wp_ff1, (size_t)ffn * d, ffn, d, sms, p.R);
    plan_gemm(p.g[SG_FF2], w.wp_ff2, (size_t)d * ffn, d, ffn, sms, p.R);
    plan_gemm(p.g[SG_HEADS], w.wp_heads, 0, NH, d, sms, p.R);
    int kb_max = 1;
    for (int i = 0; i < ACB_STEP_GEMMS; ++i) kb_max = kb_max > p.g[i].kb_per ? kb_max : p.g[i].kb_per;
    p.act_bytes = kb_max * 8 * p.R * 16;
    int dev = 0, max_smem = 0;
    ACB_CHECK_CUDA(cudaGetDevice(&dev));
    ACB_CHECK_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    int ns = (max_smem - p.act_bytes - SCRATCH_BYTES) / TILE_BYTES;
    if (ns > MAX_STAGE) ns = MAX_STAGE;
    const char* e = getenv("ACB_LM_STAGES");
    if (e && atoi(e) >= 2 && atoi(e) < ns) ns = atoi(e);
    ACB_REQUIRE(ns >= 2, "fused step: not enough shared memory for the weight ring (%d B available)", max_smem);
    p.n_stage = ns;
    p.x = b.x; p.part = b.part; p.stats = b.stats; p.a16 = (__half*)b.a16; p.h16 = (__half*)b.f16; p.logits = b.logits;
    p.kc = (__half*)b.k_cache; p.vc = (__half*)b.v_cache; p.ckc = (const __half*)b.ck_cache; p.cvc = (const __half*)b.cv_cache;
    p.seq = b.seq; p.pos = b.pos; p.bar = (unsigned*)b.bar; p.trace = nullptr;
    p.sin_pos = c.positional_embedding != 1; p.rope = c.positional_embedding >= 1; p.rope_freq = w.rope_freq;
    ACB_REQUIRE(!p.rope || w.rope_freq, "fused step: rope_freq table missing");
    p.stop_after = 1 << 30; p.max_gemms = 1 << 30;
    {   // L2 prefetch distance: the tiles all CTAs have requested ahead of the ring fill a quarter of L2, leaving the rest to the
        // KV cache and the activations (a sizing rule, not a measured optimum on the H100)
        int l2 = 0;
        ACB_CHECK_CUDA(cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev));
        p.l2_ahead = (int)((size_t)l2 / 4 / ((size_t)TILE_BYTES * (size_t)(sms > 0 ? sms : 1)));
    }
    if (const char* ea = getenv("ACB_LM_L2_AHEAD")) p.l2_ahead = atoi(ea) < 0 ? 0 : atoi(ea);
    if (const char* es = getenv("ACB_LM_STEP_STOP")) {   // bring-up aid: leave after this many grid barriers
        const int stop = atoi(es);
        if (stop >= 1) {
            // phase kinds in execution order: embed, per layer [G A G R (G A G R) G E G R], heads G; count the GEMM
            // phases among the first `stop` phases
            int n = 1, gem = 0;   // phase 0 = embed
            const int per = has_cross ? 12 : 8;
            static const int is_gemm_c[12] = {1, 0, 1, 0, 1, 0, 1, 0, 1, 0, 1, 0};
            static const int is_gemm_n[8] = {1, 0, 1, 0, 1, 0, 1, 0};
            for (int l = 0; l < c.num_layers && n < stop; ++l)
                for (int k = 0; k < per && n < stop; ++k, ++n) gem += has_cross ? is_gemm_c[k] : is_gemm_n[k];
            if (n < stop) { ++gem; ++n; }   // heads
            p.stop_after = stop; p.max_gemms = gem;
        }
    }
    L.grid = sms; L.block = BLOCK;
    L.smem = (size_t)ns * TILE_BYTES + p.act_bytes + SCRATCH_BYTES;
    L.n_phases = 1 + c.num_layers * (has_cross ? 12 : 8) + 2;
    L.cooperative = true;
    ACB_CHECK_CUDA(cudaFuncSetAttribute(lm_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.smem));
    int per_sm = 0;
    ACB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lm_step_kernel, BLOCK, L.smem));
    ACB_REQUIRE(per_sm >= 1, "fused step: the step kernel does not fit an SM (%zu B shared memory)", L.smem);
    *out = L;
    return ACB_OK;
}

int lm_step_launch(const StepLaunch& L, cudaStream_t s) {
    ACB_CHECK_CUDA(cudaMemsetAsync(L.p.bar, 0, 128, s));   // grid-barrier counter (a memset node inside the step graph)
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(L.grid); cfg.blockDim = dim3(L.block); cfg.dynamicSmemBytes = L.smem; cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = L.cooperative ? 1 : 0;
    cfg.attrs = attr; cfg.numAttrs = 1;
    ACB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, lm_step_kernel, L.p));
    return ACB_OK;
}
