// agg_kernel.cuh -- shared device helpers and the persistent MGM aggregation kernel (sm_90a).
//
// Behavioural reference (what must be reproduced bit for bit), paths under
// $REF/3rdparty/mgm_multi ($REF: the root of the s2p sources): census_tools.cc:127-153 (census),
// mgm_costvolume.cc:74-174 (cost volume), mgm_core.cc:75-124,829-1074 (MGM
// recursion, WTA, consensus), mgm_refine.h:45-90 + refine.h:40-92 (sub-pixel).
// The architecture below is ours; nothing is translated from those files.
//
// HBM layout (per view):
//   census  u64  [H][W]
//   C       u8   [H][W][DP]   popcount of the census XOR as an 8-bit code, 0xFF = +INF = label outside the
//                             pixel's range or outside the image (cost_encode / cost_decode below)
//           f32  [H][W][DP]   instead, for the "general" flavour (GEN): the other distances of the reference's
//                             table (ad, sd, ncc, btad, btsd) and / or per-pixel regularity weights (-wl / -wr)
//   L_p     f32  [H][W][DP]   one volume per scan pass p (kept separate so that the
//                             passes run concurrently and are still summed in the
//                             reference's 1-thread order 0..7)
//   Lmin_p  f32  [H][W]       per-pass vector minimum; only the band-closing scanlines are written (the next band
//                             reads them back); the per-pass LAST arg-minimum for the consensus is recomputed by the
//                             WTA kernel from L_p
// The folded layout (FOLD, DESIGN.md section 3.6) replaces the L_p volumes by the running sum S, a buffer of band-closing
// scanlines and one int16 arg-minimum plane per pass (FoldView below).
// DP = 32*LPL slots per pixel (LPL labels per lane); a warp owns one pixel, lane l owns
// slots [l*LPL, (l+1)*LPL), so every access to a pixel's vector is one fully coalesced
// 64*LPL- or 128*LPL-byte request whatever the scan direction of the pass.
//
// All float arithmetic follows the reference's operation order; the translation unit is
// compiled with -fmad=false and every fused operation below is written explicitly.
#pragma once
#include <cuda_fp16.h>
#include <type_traits>
#include <cuda_runtime.h>
#include <stdint.h>

namespace s2pb {

#define S2PB_INF __int_as_float(0x7f800000)

constexpr int kMaxPasses = 8;
constexpr int kMaxPV = 16;    // pass-views handled by one aggregation launch (2 views x 8 passes)
constexpr int kNW = 16;       // scanlines per band
constexpr int kNWC = 8;       // warps per CTA, two scanlines each
constexpr int kAggThreads = kNWC * 32;
// One CTA barrier every SECOND pixel step (volumes of 5..8 labels per lane): consecutive warps are skewed by one
// extra pixel, so that what a warp reads from its predecessor's ring was written two steps earlier and a barrier
// after every odd step separates the two; the ring is 8 deep so that a slot is not reused within that slack.
// Volumes of 4 labels per lane or fewer keep the barrier after every step.  (Chosen on the GPU the engine was first
// written for; the H100 A/B at 6 labels per lane is in DESIGN.md section 6.)
template <int LPL> struct SyncCfg {
    static constexpr bool sync2 = LPL > 4 && LPL <= 8;
    static constexpr int kRing = sync2 ? 8 : 4;      // ring slots per compute warp for handing vectors to the next warp
};
constexpr int kPublish = 8;   // a band publishes its progress every kPublish pixels

// ------------------------------------------------------------------ small helpers

__device__ __forceinline__ float fmin3f(float a, float b, float c)
{
    return fminf(fminf(a, b), c);
}
// minimum over the warp, the same value in every lane (NaN lanes are ignored, as by fminf)
__device__ __forceinline__ float warp_min_f32(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// (x, y) pairs of correctly rounded float operations: the two scanlines of a warp step together (recurse2)
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c)
{
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ int ld_acquire(const int *p)
{
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(int *p, int v)
{
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// per-lane vector load/store of LPL consecutive floats / halfs (16-byte requests when possible)
template <int LPL> __device__ __forceinline__ void ld_vec_cg(const float *p, float (&v)[LPL])
{
    if constexpr (LPL % 4 == 0) {
#pragma unroll
        for (int q = 0; q < LPL / 4; q++) {
            float4 t = __ldcg(reinterpret_cast<const float4 *>(p) + q);
            v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
        }
    } else if constexpr (LPL % 2 == 0) {
#pragma unroll
        for (int q = 0; q < LPL / 2; q++) {
            float2 t = __ldcg(reinterpret_cast<const float2 *>(p) + q);
            v[2 * q] = t.x; v[2 * q + 1] = t.y;
        }
    } else {
#pragma unroll
        for (int q = 0; q < LPL; q++) v[q] = __ldcg(p + q);
    }
}
template <int LPL> __device__ __forceinline__ void ld_vec(const float *p, float (&v)[LPL])
{
    if constexpr (LPL % 4 == 0) {
#pragma unroll
        for (int q = 0; q < LPL / 4; q++) {
            float4 t = reinterpret_cast<const float4 *>(p)[q];
            v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
        }
    } else if constexpr (LPL % 2 == 0) {
#pragma unroll
        for (int q = 0; q < LPL / 2; q++) {
            float2 t = reinterpret_cast<const float2 *>(p)[q];
            v[2 * q] = t.x; v[2 * q + 1] = t.y;
        }
    } else {
#pragma unroll
        for (int q = 0; q < LPL; q++) v[q] = p[q];
    }
}
template <int LPL> __device__ __forceinline__ void st_vec(float *p, const float (&v)[LPL])
{
    if constexpr (LPL % 4 == 0) {
#pragma unroll
        for (int q = 0; q < LPL / 4; q++)
            reinterpret_cast<float4 *>(p)[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    } else if constexpr (LPL % 2 == 0) {
#pragma unroll
        for (int q = 0; q < LPL / 2; q++) reinterpret_cast<float2 *>(p)[q] = make_float2(v[2 * q], v[2 * q + 1]);
    } else {
#pragma unroll
        for (int q = 0; q < LPL; q++) p[q] = v[q];
    }
}
// ------------------------------------------------------------------ 8-bit census cost codes
//
// The census cost volume stores one byte per slot: code = the popcount (0..127; census windows give at most 120),
// kCostInf (0xFF) = +INF.  Any code with its top bit set decodes to +INF, which lets the packed decoder find INF slots
// with one sign-replicating byte permute.  Every producer and consumer goes through the helpers below; decoding gives
// exactly (float)code.
constexpr unsigned kCostInf = 0xFFu;
constexpr int kCostMaxCode = 127;     // largest finite cost the format holds
constexpr int kCostLut = kCostMaxCode + 1;   // entries of the popcount -> cost table of the scaled census costs
// census_tools.cc:38-57,76-99: a window of side 2 (win / 2) + 1 gives side^2 - 1 code bits (at most 120 up to win 11, which the
// format holds); above 64 bits a code takes a second 64-bit word
__host__ __device__ constexpr int census_side(int win) { return 2 * (win / 2) + 1; }
__host__ __device__ constexpr int census_bits(int win) { return census_side(win) * census_side(win) - 1; }
__host__ __device__ constexpr int census_words(int win) { return census_bits(win) > 64 ? 2 : 1; }
// the two-word code (hi : lo) shifted left by one with `bit` in
__device__ __forceinline__ void census_push(uint64_t &lo, uint64_t &hi, unsigned bit) { hi = (hi << 1) | (lo >> 63); lo = (lo << 1) | bit; }
__host__ __device__ __forceinline__ unsigned cost_encode(unsigned cnt, bool finite) { return finite ? cnt : kCostInf; }
__device__ __forceinline__ unsigned char cost_encode_f(float c) { return isinf(c) ? (unsigned char)kCostInf : (unsigned char)(int)c; }
__device__ __forceinline__ float cost_decode(unsigned code) { return (code & 0x80u) ? S2PB_INF : (float)code; }
// four codes of one word (byte j = slot j) -> their values.  Per pair of slots: the halfs 0x64vv (= 1024 + v exactly) from
// one byte permute, an all-ones mask where the code is INF from a sign-replicating permute, 0x7C00 (half +INF) selected
// under it, then 1024 subtracted for both in half2 arithmetic; the f16 -> f32 conversion is the one a stored f16 needed.
// prmt.b32 in its default mode: a selector nibble with its top bit set replicates the sign of the selected byte (__byte_perm
// keeps only the low three bits of each nibble)
__device__ __forceinline__ unsigned prmt(unsigned a, unsigned b, unsigned sel)
{
    unsigned r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
    return r;
}
template <int N> __device__ __forceinline__ void cost_decode_word(unsigned w, float *c)
{
    const __half2 k1024 = __half2half2(__ushort_as_half((unsigned short)0x6400));
#pragma unroll
    for (int j = 0; j < N; j += 2) {
        const unsigned h = prmt(w, 0x6464u, j == 0 ? 0x4140u : 0x4342u);     // 0x64 b(j+1) 0x64 b(j)
        const unsigned m = prmt(w, 0u, j == 0 ? 0x9988u : 0xbbaau);          // sign of b(j), b(j+1) over their halfs
        unsigned sel = (h & ~m) | (0x7c007c00u & m);
        const __half2 v = __hsub2(*reinterpret_cast<const __half2 *>(&sel), k1024);
        c[j] = __low2float(v);
        if (j + 1 < N) c[j + 1] = __high2float(v);
    }
}
// encode a lane's LPL slots: byte e = cnt[e] where bit e of `fin` is set, else kCostInf
template <int LPL> struct CostPack { unsigned w[(LPL + 3) / 4]; };
template <int LPL> __device__ __forceinline__ CostPack<LPL> cost_pack(const unsigned (&cnt)[LPL], unsigned fin)
{
    CostPack<LPL> r;
#pragma unroll
    for (int q = 0; q < (LPL + 3) / 4; q++) {
        unsigned v = 0;
#pragma unroll
        for (int j = 0; j < 4 && 4 * q + j < LPL; j++) v |= cost_encode(cnt[4 * q + j], (fin >> (4 * q + j)) & 1u) << (8 * j);
        r.w[q] = v;
    }
    return r;
}
template <int LPL> __device__ __forceinline__ unsigned cost_code(const CostPack<LPL> &p, int e) { return (p.w[e / 4] >> (8 * (e & 3))) & 0xffu; }
template <int LPL> __device__ __forceinline__ void cost_unpack(const CostPack<LPL> &p, float (&c)[LPL])
{
#pragma unroll
    for (int q = 0; q < LPL / 4; q++) cost_decode_word<4>(p.w[q], c + 4 * q);
    if constexpr (LPL % 4 != 0) cost_decode_word<LPL % 4>(p.w[LPL / 4], c + 4 * (LPL / 4));
}
// a lane's LPL codes, widest aligned access (GLOBAL: read-only path; else a plain load, e.g. from shared memory)
template <int LPL, bool GLOBAL> __device__ __forceinline__ CostPack<LPL> ld_cost(const uint8_t *p)
{
    CostPack<LPL> r;
    if constexpr (LPL % 16 == 0) {
#pragma unroll
        for (int q = 0; q < LPL / 16; q++) {
            const uint4 t = GLOBAL ? __ldg(reinterpret_cast<const uint4 *>(p) + q) : reinterpret_cast<const uint4 *>(p)[q];
            r.w[4 * q] = t.x; r.w[4 * q + 1] = t.y; r.w[4 * q + 2] = t.z; r.w[4 * q + 3] = t.w;
        }
    } else if constexpr (LPL % 8 == 0) {
#pragma unroll
        for (int q = 0; q < LPL / 8; q++) {
            const uint2 t = GLOBAL ? __ldg(reinterpret_cast<const uint2 *>(p) + q) : reinterpret_cast<const uint2 *>(p)[q];
            r.w[2 * q] = t.x; r.w[2 * q + 1] = t.y;
        }
    } else if constexpr (LPL % 4 == 0) {
#pragma unroll
        for (int q = 0; q < LPL / 4; q++) r.w[q] = GLOBAL ? __ldg(reinterpret_cast<const unsigned *>(p) + q) : reinterpret_cast<const unsigned *>(p)[q];
    } else {
        // 1, 2, 3, 5, 6 labels per lane: a lane's codes are only 1- or 2-byte aligned
#pragma unroll
        for (int q = 0; q < (LPL + 3) / 4; q++) r.w[q] = 0;
        if constexpr (LPL % 2 == 0) {
#pragma unroll
            for (int q = 0; q < LPL / 2; q++) {
                const unsigned short t = GLOBAL ? __ldg(reinterpret_cast<const unsigned short *>(p) + q) : reinterpret_cast<const unsigned short *>(p)[q];
                r.w[q / 2] |= (unsigned)t << (16 * (q & 1));
            }
        } else {
#pragma unroll
            for (int q = 0; q < LPL; q++) r.w[q / 4] |= (unsigned)(GLOBAL ? __ldg(p + q) : p[q]) << (8 * (q & 3));
        }
    }
    return r;
}
// store a lane's LPL codes, widest aligned access
template <int LPL> __device__ __forceinline__ void st_cost(uint8_t *p, const CostPack<LPL> &v)
{
    if constexpr (LPL % 16 == 0) {
#pragma unroll
        for (int q = 0; q < LPL / 16; q++) reinterpret_cast<uint4 *>(p)[q] = make_uint4(v.w[4 * q], v.w[4 * q + 1], v.w[4 * q + 2], v.w[4 * q + 3]);
    } else if constexpr (LPL % 8 == 0) {
#pragma unroll
        for (int q = 0; q < LPL / 8; q++) reinterpret_cast<uint2 *>(p)[q] = make_uint2(v.w[2 * q], v.w[2 * q + 1]);
    } else if constexpr (LPL % 4 == 0) {
#pragma unroll
        for (int q = 0; q < LPL / 4; q++) reinterpret_cast<unsigned *>(p)[q] = v.w[q];
    } else if constexpr (LPL % 2 == 0) {
#pragma unroll
        for (int q = 0; q < LPL / 2; q++) reinterpret_cast<unsigned short *>(p)[q] = (unsigned short)(v.w[q / 2] >> (16 * (q & 1)));
    } else {
#pragma unroll
        for (int q = 0; q < LPL; q++) p[q] = (uint8_t)(v.w[q / 4] >> (8 * (q & 3)));
    }
}
// cost value of a stored code: the popcount itself (census 5x5: ratio = 1, one code word) or
// the reference's scaled cost through a kCostLut-entry table (mgm_costvolume.h:90-91)
__device__ __forceinline__ float cost_scaled(float c, const float *__restrict__ lut)
{
    if (lut != nullptr && c >= 0.f && c < (float)kCostLut) c = lut[(int)c];
    return c;
}
__device__ __forceinline__ float cost_value(unsigned code, const float *__restrict__ lut) { return cost_scaled(cost_decode(code), lut); }

// ------------------------------------------------------------------ MGM aggregation

// A scan pass in "scan coordinates": scanline s = 0..nS-1 in processing order, position
// i = 0..nI-1 along the scanline in processing order; pixel index = base + s*strideS + i*strideI.
// In these coordinates every pass of the reference's table (mgm_core.cc:884-891) has the same
// four neighbours -- A=(i-1,s) in-line, B=(i-1,s-1), Cn=(i,s-1), E=(i+1,s-1) -- listed in one of
// two orders: type 0 (passes 0-3) = A,Cn,B,E ; type 1 (passes 4-7) = E,B,Cn,A.  TSGM takes
// the first TSGM of them.
//
// Execution model.  A band = kNW (16) consecutive scanlines = one CTA of kNWC (8) warps; lanes run over
// labels.  Scanline s trails scanline s-1 by SKEW pixels (1, or 2 when the neighbour E is used).  A warp
// owns TWO adjacent scanlines: the lower one reads the upper one's last results straight from registers,
// the two pixels of a step are independent instruction streams (ILP 2), and only every second scanline
// boundary goes through a shared-memory ring to the next warp.  The CTA advances in lock step, one
// __syncthreads per pixel step.  Everything that comes from global memory -- the 8-bit cost codes of the warp's
// two scanlines (at most one 16-byte cp.async per lane and step up to 8 labels per lane) and, for the band's first scanline, the previous
// band's aggregated vectors (re-read from L2 behind a release/acquire progress counter) -- is staged into
// shared memory kStage-1 steps ahead, so no global-memory latency sits on the lock-step critical path.
// CTAs are persistent and pull (band, pass-view) items from a global queue ordered band-major, which
// keeps the chain of bands deadlock free.
struct PassDesc {
    int nS, nI;
    long long base;
    int strideS, strideI;
    int type;
    int nBands;
    const void *C;   // u8 codes (census popcounts) or float (GEN) [H][W][DP]
    const float *W;  // GEN: this view's regularity weight image (-wl / -wr), nullptr = all ones
    float *L;
    float *Lmin;     // minima of the band-closing scanlines only (read back by the next band)
    int *progress;   // [nBands] pixels of the band's last scanline visible in global memory
};
struct AggParams {
    PassDesc pv[kMaxPV];
    int nPV, maxBands;
    float P1, P2;
    int *next_item;
    const int *abort_flag;
    const float *lut;
    int general;     // 1: GEN flavour (float costs, optional per-pixel weights)
};
// The folded layout (DESIGN.md section 3.6): a launch carries one pass index and, instead of the pass volume L_p, each
// pass-view updates the running sum S of its view, keeps only its band-closing scanlines (the next band reads them) and
// records the pass's last arg-minimum per pixel for the consensus.
struct FoldView {
    float *S;        // [H][W][DP] sum of the passes so far, added in pass order as the WTA adds them
    float *Lb;       // [bands][nI][DP] L_p of each band's closing scanline, at (band, i)
    short *am;       // [H][W] the LAST slot attaining the minimum of L_p (wta_add_pass)
};
struct AggFoldParams : AggParams {
    FoldView fv[kMaxPV];
    int first;       // 1: the launch carries pass 0 (S = 0 + L_0), else S = S + L_p
};
template <bool FOLD> using AggArgs = typename std::conditional<FOLD, AggFoldParams, AggParams>::type;

// cp.async pipeline depth in pixel steps (kStage) and slots of the previous-band ring (kR0 > kStage + 1,
// because pixel 0 is staged ahead of the pipeline); shallower for the widest volumes.  (16 labels per lane would
// still fit 227 KB with 8 stages, but measured no faster: 32.7 vs 31.9 ms on the C3-like mgm_multi tile.)
template <int LPL, bool GEN = false> struct StageCfg {
    static constexpr int kStage = GEN ? ((LPL <= 4) ? 8 : (LPL <= 8) ? 4 : 2) : ((LPL <= 12) ? 8 : 2);
    static constexpr int kR0 = 2 * kStage;
};

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem)
{
    unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async4(void *smem, const void *gmem)
{
    unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(sa), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// copy NBYTES (multiple of 16) from global to shared with the whole warp
template <int NBYTES> __device__ __forceinline__ void warp_cp_async(void *smem, const void *gmem, int lane)
{
    constexpr int CH = NBYTES / 16;
#pragma unroll
    for (int q = 0; q < (CH + 31) / 32; q++) {
        int c = lane + 32 * q;
        if (CH % 32 == 0 || c < CH) cp_async16((char *)smem + 16 * c, (const char *)gmem + 16 * c);
    }
}
// x / 3 with two fmas: bit-identical to IEEE division for every finite x >= 0
// (exhaustively verified on the CPU: tests/test_host_logic.py::test_div3_trick)
__device__ __forceinline__ float div3_exact(float x)
{
    const float r3 = 0.3333333432674407958984375f;   // RN(1/3)
    float q0 = x * r3;
    float r = fmaf(-3.0f, q0, x);
    return fmaf(r, r3, q0);
}

template <int LPL> struct NbVec {
    float v[LPL];
    float l, r;   // slots just left / right of this lane's, from the neighbouring lanes (INF at the ends)
    float m;      // minimum of the whole vector
};
template <int LPL> __device__ __forceinline__ void fill_edges(NbVec<LPL> &n, int lane)
{
    float l = __shfl_up_sync(0xffffffffu, n.v[LPL - 1], 1);
    float r = __shfl_down_sync(0xffffffffu, n.v[0], 1);
    n.l = (lane == 0) ? S2PB_INF : l;
    n.r = (lane == 31) ? S2PB_INF : r;
}
// A neighbour vector's message: its contribution to every slot e of a pixel that takes it as a neighbour, with unit
// weights (update_costW, mgm_core.cc:92-121): M[e] = min(v[e], min(v[e-1], v[e+1]) + P1, min(v) + P2) - min(v).  It
// depends on the vector alone (slots outside the vector's range hold +INF), so the census flavours compute it once,
// where the vector is produced, and hand it to all its consumers; the operations are those of recurse2's `term`.
// n.v, n.l, n.r, n.m in; the message out in n.v.
template <int LPL> __device__ __forceinline__ void nb_message(NbVec<LPL> &n, float P1, float P2)
{
    const float q = __fadd_rn(n.m, P2), negm = -n.m;
    float M[LPL];
#pragma unroll
    for (int e = 0; e < LPL; e++) {
        const float a = (e == 0) ? n.l : n.v[e - 1], b = (e == LPL - 1) ? n.r : n.v[e + 1];
        M[e] = __fadd_rn(fmin3f(n.v[e], __fadd_rn(fminf(a, b), P1), q), negm);
    }
#pragma unroll
    for (int e = 0; e < LPL; e++) n.v[e] = M[e];
}

// shared memory carve-up of one CTA (floats first, then cost codes; every block 16-byte aligned)
template <int LPL, bool GEN = false> struct AggSmem {
    static constexpr int DP = 32 * LPL;
    static constexpr int kStage = StageCfg<LPL, GEN>::kStage, kR0 = StageCfg<LPL, GEN>::kR0;
    static constexpr size_t kCostBytes = GEN ? sizeof(float) : sizeof(uint8_t);
    static constexpr int kRing = SyncCfg<LPL>::kRing;
    static constexpr size_t ring_off = 0;                                            // float [kNWC][kRing][DP]
    static constexpr size_t ringm_off = ring_off + sizeof(float) * kNWC * kRing * DP; // float [kNWC][kRing]  (GEN: minima)
    static constexpr size_t r0_off = ringm_off + (GEN ? sizeof(float) * kNWC * kRing : 0);   // float [kR0][DP]   previous band
    static constexpr size_t r0m_off = r0_off + sizeof(float) * kR0 * DP;              // float [kR0]
    static constexpr size_t cst_off = r0m_off + sizeof(float) * kR0;                  // u8 | float [kNW][kStage][DP]
    static constexpr size_t wst_off = cst_off + kCostBytes * kNW * kStage * DP;       // float [kNW][kStage]  (GEN: weights)
    static constexpr size_t bytes = wst_off + (GEN ? sizeof(float) * kNW * kStage : 0);
};

// smem address (32-bit, shared state space) helpers for cp.async
__device__ __forceinline__ void cp_async16_s(unsigned sa, const void *gmem)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async4_s(unsigned sa, const void *gmem)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(sa), "l"(gmem) : "memory");
}
template <int NBYTES> __device__ __forceinline__ void warp_cp_async_s(unsigned sa, const char *gmem, int lane)
{
    constexpr int CH = NBYTES / 16;
#pragma unroll
    for (int q = 0; q < (CH + 31) / 32; q++) {
        int c = lane + 32 * q;
        if (CH % 32 == 0 || c < CH) cp_async16_s(sa + 16 * c, gmem + 16 * c);
    }
}

// FOLD: one pixel's pass vector L (minimum m) into the running sum S at out: S = 0 + L_0 for pass 0, S + L_p after it -- the
// additions and their order are those of wta_add_pass, so S after pass p is the WTA's running sum -- and the LAST slot attaining m
// into *am, wta_add_pass's rule (slot lane*LPL + e).  S is read here, after the recursion: held across it, it made the widest and
// the float-cost instantiations spill.
template <int LPL>
__device__ __forceinline__ void fold_store(float *out, short *am, const float (&L)[LPL], float m, int first, int lane)
{
    float t[LPL];
    if (first) {
#pragma unroll
        for (int e = 0; e < LPL; e++) t[e] = 0.f;
    } else ld_vec_cg<LPL>(out, t);
    int a = -1;
#pragma unroll
    for (int e = 0; e < LPL; e++) {
        t[e] = __fadd_rn(t[e], L[e]);
        if (L[e] == m) a = lane * LPL + e;
    }
    st_vec<LPL>(out, t);
    a = __reduce_max_sync(0xffffffffu, a);
    if (lane == 0) *am = (short)a;
}

template <int LPL, int TSGM, int TYPE, bool SCALED, bool GEN, bool FOLD>
__device__ __forceinline__ void run_band(const PassDesc &pd, const FoldView &fv, int first, int band, float P1, float P2,
                                         const float *__restrict__ lut, const int *abort_flag, unsigned char *smem)
{
    constexpr int DP = 32 * LPL;
    constexpr bool useA = (TYPE == 0) ? true : (TSGM == 4);
    constexpr bool useCn = (TYPE == 0) ? (TSGM >= 2) : (TSGM >= 3);
    constexpr bool useB = (TYPE == 0) ? (TSGM >= 3) : (TSGM >= 2);
    constexpr bool useE = (TYPE == 0) ? (TSGM == 4) : true;
    constexpr bool usePrev = useCn || useB || useE;
    // MSG (census flavours): the registers and the ring between warps hold each vector's message (nb_message) instead of
    // the vector.  GEN scales the penalties by the current pixel's weight, so its consumers compute their terms.
    constexpr bool MSG = !GEN;
    constexpr int SKEW = useE ? 2 : 1;    // scanline s trails scanline s-1 by SKEW pixels
    constexpr int LEAD = useE ? 1 : 0;    // newest previous-scanline pixel needed at position i is i+LEAD
    constexpr int U = useE ? 3 : 2;       // window / history registers rotate with period U: the step loop is unrolled by U
    using SM = AggSmem<LPL, GEN>;
    using CT = typename std::conditional<GEN, float, uint8_t>::type;     // stored cost element
    constexpr int kStage = SM::kStage, kR0 = SM::kR0, S = kStage - 1, kRing = SM::kRing;
    constexpr bool SYNC2 = SyncCfg<LPL>::sync2;
    constexpr int WSK = SYNC2 ? 2 * SKEW + 1 : 2 * SKEW;   // pixels by which a warp's upper scanline trails the previous warp's
    constexpr int CB = DP * (int)sizeof(CT);   // bytes of one pixel's cost vector
    constexpr int CH = CB / 16;                // ... in 16-byte chunks

    const int nI = pd.nI;
    const int nsteps = (nI + (kNWC - 1) * WSK + SKEW + U - 1) / U * U;
    const int lane = threadIdx.x & 31, k = threadIdx.x >> 5;

    // ---- this warp's two scanlines: A (upper) and B = A + 1
    const int sA = band * kNW + 2 * k;
    const bool liveA = sA < pd.nS, liveB = sA + 1 < pd.nS;
    const long long strideI = pd.strideI;
    const bool prevA = usePrev && liveA && sA > 0;           // scanline A has a previous scanline (B always has A)
    const bool from_r0 = (k == 0);                           // ... which belongs to the previous band
    const bool publish = liveB && (k == kNWC - 1) && (sA + 2 < pd.nS);
    const long long rowbaseA = pd.base + (long long)sA * pd.strideS;

    const unsigned smem_s = (unsigned)__cvta_generic_to_shared(smem);
    float *ring = reinterpret_cast<float *>(smem + SM::ring_off);
    float *ringm = reinterpret_cast<float *>(smem + SM::ringm_off);
    float *myring = ring + (size_t)k * kRing * DP + lane * LPL;
    float *myringm = ringm + k * kRing;
    const float *srcring = (from_r0 ? reinterpret_cast<float *>(smem + SM::r0_off) : ring + (size_t)(k - 1) * kRing * DP) + lane * LPL;
    const float *srcringm = from_r0 ? reinterpret_cast<float *>(smem + SM::r0m_off) : ringm + (k - 1) * kRing;
    const int srcmask = from_r0 ? (kR0 - 1) : (kRing - 1);
    const CT *cstA = reinterpret_cast<CT *>(smem + SM::cst_off) + (size_t)(2 * k) * kStage * DP + lane * LPL;
    const CT *cstB = cstA + kStage * DP;
    const float *wstA = reinterpret_cast<float *>(smem + SM::wst_off) + (2 * k) * kStage, *wstB = wstA + kStage;   // GEN only
    const bool weighted = GEN && pd.W != nullptr;

    // ---- staging cursors.  Costs: lanes 0-15 copy scanline A, lanes 16-31 scanline B, 16-byte pieces.
    const int rsel = lane >> 4, q16 = lane & 15;
    const bool live_st = rsel ? liveB : liveA;
    const char *csrc = reinterpret_cast<const char *>(pd.C) + (rowbaseA + (long long)rsel * pd.strideS) * CB + 16 * q16;
    const long long cstep = strideI * CB;
    const unsigned cdst = smem_s + (unsigned)SM::cst_off + (unsigned)((2 * k + rsel) * kStage * CB + 16 * q16);
    const float *wsrc = weighted ? pd.W + rowbaseA + (long long)rsel * pd.strideS : nullptr;
    const unsigned wdst = smem_s + (unsigned)SM::wst_off + (unsigned)((2 * k + rsel) * kStage * 4);
    int jc = 0;                                               // next pixel of my scanline to stage
    //      previous band's last scanline (warp 0 only)
    const bool stage_prev = prevA && from_r0;
    const long long prevbase = rowbaseA - pd.strideS;
    // (FOLD: the previous band's closing scanline is stored contiguously in the boundary buffer)
    const char *psrc = FOLD ? reinterpret_cast<const char *>(fv.Lb + (long long)(band > 0 ? band - 1 : 0) * nI * DP)
                            : reinterpret_cast<const char *>(pd.L + prevbase * DP);
    const float *pmsrc = pd.Lmin + prevbase;
    const long long lstepb = (FOLD ? 1 : strideI) * (DP * 4);
    const unsigned r0_s = smem_s + (unsigned)SM::r0_off, r0m_s = smem_s + (unsigned)SM::r0m_off;
    const int *prev_progress = (band > 0) ? pd.progress + (band - 1) : nullptr;
    int jp = 0, avail = 0;

    auto stage_cost = [&]() {            // stage pixel jc of my scanline's costs
        if (live_st && jc < nI) {
            const unsigned d = cdst + (unsigned)((jc & (kStage - 1)) * CB);
#pragma unroll
            for (int q = 0; q < (CH + 15) / 16; q++)
                if (CH % 16 == 0 || q16 + 16 * q < CH) cp_async16_s(d + 256 * q, csrc + 256 * q);
            csrc += cstep;
            if (weighted) {
                if (q16 == 0) cp_async4_s(wdst + (unsigned)((jc & (kStage - 1)) * 4), wsrc);
                wsrc += strideI;
            }
        }
        jc++;
    };
    auto stage_prevband = [&]() {        // (warp 0) stage pixel jp of the previous band's last scanline
        if (stage_prev) {
            if (jp < nI) {
                int spins = 0;
                while (avail < jp + 1) {
                    avail = ld_acquire(prev_progress);
                    if (((++spins) & 1023) == 0 && *(volatile const int *)abort_flag) break;
                }
                const unsigned slot = (unsigned)(jp & (kR0 - 1));
                warp_cp_async_s<DP * 4>(r0_s + slot * (DP * 4), psrc, lane);
                if (lane == 0) cp_async4_s(r0m_s + slot * 4, pmsrc);
                psrc += lstepb;
                pmsrc += strideI;
            }
            jp++;
        }
    };

    // ---- global output cursors
    const long long lstep = strideI * DP;                    // floats per pixel step along the scanline
    float *outA = (FOLD ? fv.S : pd.L) + rowbaseA * DP + lane * LPL;      // FOLD: the running sum S instead of L_p
    float *outB = outA + (long long)pd.strideS * DP;
    float *lminB = pd.Lmin + rowbaseA + pd.strideS;          // only the band's last scanline publishes its minima
    float *lbB = FOLD ? fv.Lb + (long long)band * nI * DP + lane * LPL : nullptr;   // FOLD: ... and its vectors
    short *amA = FOLD ? fv.am + rowbaseA : nullptr, *amB = FOLD ? amA + pd.strideS : nullptr;

    auto fetch_prev = [&](int j, NbVec<LPL> &dst) {
        const int slot = j & srcmask;
        ld_vec<LPL>(srcring + slot * DP, dst.v);
        if (!MSG || from_r0) {         // the previous band's vectors come from HBM as L: warp 0 forms their messages
            dst.m = srcringm[slot];
            fill_edges<LPL>(dst, lane);
            if (MSG) nb_message<LPL>(dst, P1, P2);
        }
    };
    auto load_cost = [&](const CT *p, float (&c)[LPL]) {
        if constexpr (GEN) {
            ld_vec<LPL>(p, c);
        } else {
            cost_unpack<LPL>(ld_cost<LPL, false>(p), c);
            if (SCALED) {
#pragma unroll
                for (int e = 0; e < LPL; e++)
                    if (c[e] >= 0.f && c[e] < (float)kCostLut) c[e] = lut[(int)c[e]];   // an idle scanline reads unstaged shared memory: never index with it
            }
        }
    };
    // L = C + (sum of the neighbours' terms) / TSGM in the reference's order; border pixels keep L = C.
    // The recursion runs for the warp's two scanlines at once: the float adds / multiplies / fmas of scanline A and
    // scanline B are written as (A, B) pairs (add2 / mul2 / fma2), each half rounding like the scalar operation, so
    // that the two independent chains interleave.  (a*, b*) = neighbours of A, of B: their messages (MSG), else vectors.
    auto recurse2 = [&](const float (&cA)[LPL], const float (&cB)[LPL],
                        const NbVec<LPL> &aA, const NbVec<LPL> &aB, const NbVec<LPL> &aC, const NbVec<LPL> &aE,
                        const NbVec<LPL> &bA, const NbVec<LPL> &bB, const NbVec<LPL> &bC, const NbVec<LPL> &bE,
                        bool borderA, bool borderB, const float2 wv, float (&LA)[LPL], float (&LB)[LPL], auto interior_c) {
        constexpr bool INTERIOR = decltype(interior_c)::value;     // both pixels are interior: no border select
        const float2 P1v = make_float2(P1, P1), P2v = make_float2(P2, P2);
        const float2 mA = make_float2(aA.m, bA.m), mB = make_float2(aB.m, bB.m), mC = make_float2(aC.m, bC.m), mE = make_float2(aE.m, bE.m);
        // GEN: the penalties are scaled by the current pixel's weight w (update_costW, mgm_core.cc:93-114).  How
        // `x + P*w` rounds in the reference build (gcc -O3 -march=native: one fma, or the product hoisted out of the
        // label loop and then added) was pinned against the binary: the P2 term of every neighbour and the P1 term
        // of the 3rd / 4th neighbour are fmas, the P1 term of the 1st / 2nd is mul + add (oracle/mgm_oracle.c,
        // orc_fma_mask).  With w = 1 all of these equal the unweighted x + P.
        const float2 P1w = GEN ? make_float2(__fmul_rn(P1, wv.x), __fmul_rn(P1, wv.y)) : P1v;
        auto qof = [&](const float2 m) { return GEN ? fma2(P2v, wv, m) : add2(m, P2v); };
        const float2 qA = qof(mA), qB = qof(mB), qC = qof(mC), qE = qof(mE);
        const float2 nA = make_float2(-mA.x, -mA.y), nB = make_float2(-mB.x, -mB.y), nC = make_float2(-mC.x, -mC.y), nE = make_float2(-mE.x, -mE.y);
        // order of the neighbours in the reference's list: type 0 = A, Cn, B, E ; type 1 = E, B, Cn, A
        constexpr int ordA = (TYPE == 0) ? 0 : 3, ordC = (TYPE == 0) ? 1 : 2, ordB = (TYPE == 0) ? 2 : 1, ordE = (TYPE == 0) ? 3 : 0;
        auto term = [&](const NbVec<LPL> &na, const NbVec<LPL> &nb, int e, const float2 q, const float2 negm, auto ord_c) {
            if constexpr (MSG) return make_float2(na.v[e], nb.v[e]);
            constexpr bool FMA1 = GEN && decltype(ord_c)::value >= 2;
            const float la = (e == 0) ? na.l : na.v[e - 1], ra = (e == LPL - 1) ? na.r : na.v[e + 1];
            const float lb = (e == 0) ? nb.l : nb.v[e - 1], rb = (e == LPL - 1) ? nb.r : nb.v[e + 1];
            const float2 mn = make_float2(fminf(la, ra), fminf(lb, rb));
            const float2 v1 = FMA1 ? fma2(P1v, wv, mn) : add2(mn, P1w);
            const float2 t = make_float2(fmin3f(na.v[e], v1.x, q.x), fmin3f(nb.v[e], v1.y, q.y));
            return add2(t, negm);
        };
        using oA = std::integral_constant<int, ordA>; using oB = std::integral_constant<int, ordB>;
        using oC = std::integral_constant<int, ordC>; using oE = std::integral_constant<int, ordE>;
        const float2 half2v = make_float2(0.5f, 0.5f), quart = make_float2(0.25f, 0.25f);
        const float r3 = 0.3333333432674407958984375f;
        const float2 r3v = make_float2(r3, r3), m3v = make_float2(-3.0f, -3.0f);
#pragma unroll
        for (int e = 0; e < LPL; e++) {
            float2 acc;
            if constexpr (TYPE == 0) {
                acc = term(aA, bA, e, qA, nA, oA{});
                if (TSGM == 2) acc = mul2(acc, half2v);
                if (useCn) { float2 tt = term(aC, bC, e, qC, nC, oC{}); if (TSGM == 2) tt = mul2(tt, half2v); acc = add2(acc, tt); }
                if (useB)  acc = add2(acc, term(aB, bB, e, qB, nB, oB{}));
                if (useE)  acc = add2(acc, term(aE, bE, e, qE, nE, oE{}));
            } else {
                acc = term(aE, bE, e, qE, nE, oE{});
                if (TSGM == 2) acc = mul2(acc, half2v);
                if (useB)  { float2 tt = term(aB, bB, e, qB, nB, oB{}); if (TSGM == 2) tt = mul2(tt, half2v); acc = add2(acc, tt); }
                if (useCn) acc = add2(acc, term(aC, bC, e, qC, nC, oC{}));
                if (useA)  acc = add2(acc, term(aA, bA, e, qA, nA, oA{}));
            }
            if constexpr (TSGM == 3) {            // exact x/3, see div3_exact
                const float2 q0 = mul2(acc, r3v);
                const float2 rr = fma2(m3v, q0, acc);
                acc = fma2(rr, r3v, q0);
            }
            if constexpr (TSGM == 4) acc = mul2(acc, quart);
            const float la = __fadd_rn(cA[e], acc.x), lb = __fadd_rn(cB[e], acc.y);
            LA[e] = (!INTERIOR && borderA) ? cA[e] : la;
            LB[e] = (!INTERIOR && borderB) ? cB[e] : lb;
        }
    };
    auto vec_min = [&](const float (&L)[LPL]) {
        float lm = L[0];
#pragma unroll
        for (int e = 1; e < LPL; e++) lm = fminf(lm, L[e]);
        return warp_min_f32(lm);
    };

    NbVec<LPL> x0, x1, x2, h0, h1, h2, wAB;                   // window on A's previous scanline, A's last results, B's last result
                                                              // (MSG: their messages)
#pragma unroll
    for (int e = 0; e < LPL; e++) x0.v[e] = x1.v[e] = x2.v[e] = h0.v[e] = h1.v[e] = h2.v[e] = wAB.v[e] = 0.f;
    x0.l = x0.r = x0.m = x1.l = x1.r = x1.m = x2.l = x2.r = x2.m = 0.f;
    h0.l = h0.r = h0.m = h1.l = h1.r = h1.m = h2.l = h2.r = h2.m = wAB.l = wAB.r = wAB.m = 0.f;

    // prologue: S groups in flight; group g holds costs(g) and previous-band pixel g+LEAD (+ pixel 0 when LEAD = 1)
    if (LEAD == 1) stage_prevband();
#pragma unroll 1
    for (int g = 0; g < S; g++) { stage_cost(); stage_prevband(); cp_async_commit(); }

    // One lock-step pixel step.  Roles at step t: (xB, xC, xE) = window on A's previous scanline at A's
    // pixel-1, pixel, pixel+1; hNew = A's result of U steps ago (B's "B" neighbour; overwritten with A's new
    // result at the end of the step), hC / hE = A's results of U-1.. / 1 steps ago.
    // FAST: both scanlines are live and at interior pixels (warp-uniform), which removes every activity / border /
    // end-of-line predicate from the step; the slow variant handles ramp-up, ramp-down and the image border.
    auto step = [&](auto fast_c, const int t, NbVec<LPL> &xB, NbVec<LPL> &xC, NbVec<LPL> &xE, NbVec<LPL> &hNew, NbVec<LPL> &hC, NbVec<LPL> &hE) {
        constexpr bool FAST = decltype(fast_c)::value;
        const int iA = t - k * WSK, iB = iA - SKEW;
        const bool actA = FAST || (liveA && iA >= 0 && iA < nI), actB = FAST || (liveB && iB >= 0 && iB < nI);
        NbVec<LPL> &inlineA = useE ? hE : hC;                 // A's result of the previous step
        if (FAST || iA - rsel * SKEW >= 0) stage_cost();      // my scanline is at pixel jc - S: stage pixel jc
        if (FAST || iA >= 0) stage_prevband();
        cp_async_commit();
        if (actA || actB) {
            cp_async_wait<S>();                               // the groups of this step's pixels have landed
            __syncwarp();
            float cA[LPL], cB[LPL], LA[LPL], LB[LPL];
#pragma unroll
            for (int e = 0; e < LPL; e++) cA[e] = cB[e] = 0.f;
            if (actA) load_cost(cstA + (iA & (kStage - 1)) * DP, cA);     // an idle scanline's slot is not staged yet
            if (actB) load_cost(cstB + (iB & (kStage - 1)) * DP, cB);
            if (FAST) {
                if (useE) fetch_prev(iA + 1, xE); else fetch_prev(iA, xC);
            } else if (prevA && actA) {
                if (useE) { if (iA == 0) fetch_prev(0, xC); if (iA + 1 < nI) fetch_prev(iA + 1, xE); }
                else fetch_prev(iA, xC);
            }
            const bool borderA = (sA == 0) || (iA == 0) || (iA == nI - 1);
            const bool borderB = (iB == 0) || (iB == nI - 1);
            float2 wv = make_float2(1.f, 1.f);
            if (GEN) { if (weighted) { if (actA) wv.x = wstA[iA & (kStage - 1)]; if (actB) wv.y = wstB[iB & (kStage - 1)]; } }
            recurse2(cA, cB, inlineA, xB, xC, xE, wAB, hNew, hC, hE, borderA, borderB, wv, LA, LB, fast_c);
            const float mAm = vec_min(LA), mBm = vec_min(LB);
            if (actA) {
#pragma unroll
                for (int e = 0; e < LPL; e++) hNew.v[e] = LA[e];
                hNew.m = mAm;
                fill_edges<LPL>(hNew, lane);
                if (MSG) nb_message<LPL>(hNew, P1, P2);
                if constexpr (FOLD) fold_store<LPL>(outA, amA, LA, mAm, first, lane);
                else st_vec<LPL>(outA, LA);
                outA += lstep;
                if (FOLD) amA += strideI;
            }
            if (actB) {
#pragma unroll
                for (int e = 0; e < LPL; e++) wAB.v[e] = LB[e];
                wAB.m = mBm;
                if (MSG && (useA || usePrev)) {     // B's message, for its next step (useA) and the next warp's ring
                    fill_edges<LPL>(wAB, lane);
                    nb_message<LPL>(wAB, P1, P2);
                } else if (useA) {
                    fill_edges<LPL>(wAB, lane);
                }
                if (usePrev) st_vec<LPL>(myring + (iB & (kRing - 1)) * DP, MSG ? wAB.v : LB);
                if constexpr (FOLD) {
                    fold_store<LPL>(outB, amB, LB, mBm, first, lane);
                    if (publish) st_vec<LPL>(lbB + (long long)iB * DP, LB);
                } else st_vec<LPL>(outB, LB);
                outB += lstep;
                if (FOLD) amB += strideI;
                if (!MSG && lane == 0 && usePrev) myringm[iB & (kRing - 1)] = mBm;
                if (publish) {
                    if (lane == 0) *lminB = mBm;
                    lminB += strideI;
                    if (((iB + 1) % kPublish) == 0 || iB == nI - 1) {
                        __syncwarp();
                        if (lane == 0) st_release(pd.progress + band, iB + 1);
                    }
                }
            }
        }
        if (!SYNC2 || (t & 1)) __syncthreads();
        else __syncwarp();      // the staging slot the lanes just read is overwritten by the next step's cp.async
    };
    // a step is FAST for this warp when A is at an interior pixel with B one SKEW behind, also interior
    const bool can_fast = liveA && liveB && prevA;
    const int fast_lo = k * WSK + SKEW + 1, fast_hi = k * WSK + nI - 2;     // t range: iB >= 1 and iA <= nI-2

    // every warp runs its own three loops -- ramp-up, interior, ramp-down -- so that the interior steps carry no
    // fast / slow test and the compiler keeps one register assignment through the interior loop; the barrier sequence
    // is the same for all warps
    auto group = [&](auto fast_c, const int t) {
        if constexpr (U == 2) {
            step(fast_c, t, x1, x0, x2, h0, h1, h2);
            step(fast_c, t + 1, x0, x1, x2, h1, h0, h2);
        } else {
            step(fast_c, t, x1, x2, x0, h0, h1, h2);
            step(fast_c, t + 1, x2, x0, x1, h1, h2, h0);
            step(fast_c, t + 2, x0, x1, x2, h2, h0, h1);
        }
    };
    int ta = nsteps, tb = nsteps;                          // [ta, tb): groups whose U steps are all interior for this warp
    if (can_fast) {
        ta = (fast_lo + U - 1) / U * U;
        tb = (fast_hi + 1) / U * U;
        if (tb < ta) tb = ta;
        if (ta > nsteps) ta = tb = nsteps;
    }
    int t = 0;
    for (; t < ta; t += U) group(std::false_type{}, t);
    for (; t < tb; t += U) group(std::true_type{}, t);
    for (; t < nsteps; t += U) group(std::false_type{}, t);
    cp_async_wait<0>();
}

// Register cap and resident CTAs per SM.  Up to 4 labels per lane two CTAs fit at 112 registers; for 5..8 labels per
// lane (160..256 labels) a cap of 128 registers still holds two CTAs (8 x 32 x 128 x 2 = the whole register file)
// with no or few spills, which doubles the warps available to hide the lock-step latency; the 4-neighbour recursion
// at 8 labels per lane and the widest volumes keep one CTA with all the registers they want.
#ifndef S2PB_WIDE_TWO_CTAS
#define S2PB_WIDE_TWO_CTAS 0   /* chosen on the GPU the engine was first written for (two wide CTAs per SM left no room for the
                                  WTA CTAs of the next tile in flight); the H100 A/B is in DESIGN.md section 6 */
#endif
template <int LPL, int TSGM> struct AggOcc {
    static constexpr bool two_wide = S2PB_WIDE_TWO_CTAS && (LPL <= 6 || (LPL == 8 && TSGM <= 3));
    static constexpr int regs = (LPL <= 4) ? 112 : (two_wide ? 128 : 255);
    static constexpr int ctas = (regs <= 128) ? 2 : 1;
};
// FOLD: the folded layout (AggFoldParams): one pass index per launch, S, boundary buffer and arg-minimum plane instead of L_p
template <int LPL, int TSGM, bool SCALED, bool GEN, bool FOLD = false>
__global__ void __launch_bounds__(kAggThreads) __maxnreg__((AggOcc<LPL, TSGM>::regs)) aggregate_kernel(const __grid_constant__ AggArgs<FOLD> P)
{
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int s_item;
    const int total = P.maxBands * P.nPV;
    for (;;) {
        if (threadIdx.x == 0) s_item = atomicAdd(P.next_item, 1);
        __syncthreads();
        const int item = s_item;
        __syncthreads();
        if (item >= total) return;
        const int band = item / P.nPV, pvi = item - band * P.nPV;
        const PassDesc &pd = P.pv[pvi];
        if (band >= pd.nBands) continue;
        if constexpr (FOLD) {
            if (pd.type == 0) run_band<LPL, TSGM, 0, SCALED, GEN, true>(pd, P.fv[pvi], P.first, band, P.P1, P.P2, P.lut, P.abort_flag, smem);
            else run_band<LPL, TSGM, 1, SCALED, GEN, true>(pd, P.fv[pvi], P.first, band, P.P1, P.P2, P.lut, P.abort_flag, smem);
        } else {
            const FoldView none{};
            if (pd.type == 0) run_band<LPL, TSGM, 0, SCALED, GEN, false>(pd, none, 0, band, P.P1, P.P2, P.lut, P.abort_flag, smem);
            else run_band<LPL, TSGM, 1, SCALED, GEN, false>(pd, none, 0, band, P.P1, P.P2, P.lut, P.abort_flag, smem);
        }
    }
}

}  // namespace s2pb
