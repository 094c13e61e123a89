// Tensor-core SYRK / TN-GEMM for sm_90a:  C[i,j] = beta*C[i,j] + alpha * sum_k SA[k,i]*SB[k,j]
//
// This is LinearRegressor::learn's "At * A" (reference verbose_solver.hpp:67, regressors.hpp:208) with
// A^T b folded in as extra columns (SA == SB, upper-triangle tiles only), the trailing update of the blocked
// Cholesky that replaces PartialPivLU (verbose_solver.hpp:89), and -- with two different operands -- the
// product S P of the conjugate-gradient route (sd_cg.cu).  S is row-major [K x NJ] -- one sample per row, exactly
// as the optimiser stacks the feature rows (superviseddescent.hpp:186-189) -- so BOTH operands are "MN-major"
// (the contraction index K is the slow one).  wgmma reads 32-bit (TF32) operands from shared memory only
// K-major, so the raw tiles that the TMA brings in are transposed in shared memory by a transform warpgroup,
// which splits them into hi / lo at the same time: no transposed or split copy of A exists in HBM.
//
// Precision: TF32 keeps 10 mantissa bits.  passes == 3 runs the 3xTF32 split
//     a = hi + lo,  lo = rna_tf32(a - hi);   a_i*a_j ~= hi_i*hi_j + hi_i*lo_j + lo_i*hi_j
// (relative error ~2^-21 per product, fp32 accumulation); hi is the raw value as the tensor core truncates it,
// or rna_tf32(a) (unbiased split).  passes == 1 is a single TF32 pass on the raw operand.
//
// Accumulation: the chain of accumulating MMAs is cut every KC = 128 samples: each chunk starts a fresh
// accumulator (scale-d = 0) and the consumer warps fold the finished chunk into running sums held in registers
// with round-to-nearest adds, so the MMA chain's error does not grow with the length of the contraction; the fp32 fold over
// K / 128 chunks does, roughly like the square root of the number of chunks (DESIGN 4.2).
//
// Kernel shape (persistent, one CTA per SM, 512 threads): see syrk_wgmma_kernel below.
#include "sd_internal.cuh"

#include <cuda.h>

#include <cstring>
#include <vector>

namespace {

constexpr int BM = 128;          // rows of C per tile   (operand "A": columns i of S), two consumer warpgroups of 64 rows
constexpr int BK = 16;           // samples (rows of S) per pipeline stage
constexpr int BOX_COLS = 32;     // TMA box: 32 columns x BK rows, unswizzled
constexpr int BOX_BYTES = BOX_COLS * 4 * BK;              // 2 KB
constexpr int A_BLOCKS = BM / BOX_COLS;                   // 4
constexpr int RAW_A_BYTES = A_BLOCKS * BOX_BYTES;         // 8 KB
constexpr int KM_A_BYTES = BM * BK * 4;                   // one K-major copy of the A tile (8 KB)
constexpr int RAW_STAGES = 4;
constexpr int PIPE_BYTES = 200 * 1024;                    // shared memory of both pipelines
constexpr int MAX_KM_STAGES = 6;
constexpr int KC_STAGES = 8;     // pipeline stages per accumulation chunk: KC = 8 * BK = 128 samples

// The kernel is compiled for BN = 128 (tiles of 128 columns: the Gram, the trailing updates) and for a narrow "B" operand of
// BN = 64 columns (a single tile column: the skinny product C[MI x <=64] = SA^T SB of the CG route, bound by the read of SA).
template <int BN>
struct TcCfg {
    static constexpr int B_BLOCKS = BN / BOX_COLS;
    static constexpr int RAW_B_BYTES = B_BLOCKS * BOX_BYTES;
    static constexpr int RAW_BYTES = RAW_A_BYTES + RAW_B_BYTES;                   // one TMA stage
    static constexpr int KM_B_BYTES = BN * BK * 4;
    static constexpr int KM_HALF = KM_A_BYTES + KM_B_BYTES;                       // hi (or lo) of A and B
    static constexpr int KM_BYTES = 2 * KM_HALF;                                  // hi + lo: 32 KB for BN = 128
    static constexpr int KM_STAGES = (PIPE_BYTES - RAW_STAGES * RAW_BYTES) / KM_BYTES < MAX_KM_STAGES
                                         ? (PIPE_BYTES - RAW_STAGES * RAW_BYTES) / KM_BYTES : MAX_KM_STAGES;
    static constexpr int BAR_OFF = RAW_STAGES * RAW_BYTES + KM_STAGES * KM_BYTES;
    static constexpr int SMEM_BYTES = BAR_OFF + 1024 /*barriers*/ + 1024 /*align*/;
    static constexpr int NV = BN / 2;                                             // accumulator registers per consumer thread
    static_assert(KM_STAGES >= 2, "pipeline depth");
};

// super-tile for L2 reuse: tiles that run concurrently share (GI*128 + GJ*128) operand columns
constexpr int GI = 12, GJ = 12;

// ---- PTX wrappers ----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// bounded wait: a protocol bug must trap (context error), never hang the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 8000000000LL) __trap();
    }
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1)
{
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// One lane of a converged warp (cute::elect_one_sync): the compiler knows the guarded region runs on a single thread
__device__ __forceinline__ bool elect_one_sync()
{
    uint32_t pred = 0;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(pred));
    return pred != 0;
}

// explicit shared-space accesses: the tile pointers come from integer arithmetic on the dynamic shared-memory base, so
// the compiler would otherwise emit generic LD/ST
__device__ __forceinline__ float lds32(uint32_t addr)
{
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const float4& v)
{
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

__device__ __forceinline__ float trunc_tf32(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }
// rna_tf32 of a finite value (what cvt.rna.tf32.f32 returns): round the magnitude to 10 mantissa bits, ties away from zero
__device__ __forceinline__ float rna_tf32_bits(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }
// the same value as far as the tensor core is concerned (it ignores the low 13 bits of a TF32 operand)
__device__ __forceinline__ float round_operand(float x) { return __uint_as_float(__float_as_uint(x) + 0x1000u); }

// wgmma shared-memory descriptor, K-major operand without swizzle: 8-row x 16-byte core matrices stored as 128 contiguous bytes.
//   start [0,14), LBO [16,30) = byte distance between core matrices adjacent along K, SBO [32,46) = byte distance between
//   adjacent 8-row groups along M / N, layout type [62,64) = 0 (no swizzle); all in 16-byte units.
// Layout used here for a tile of R rows x BK samples: core matrix (row group g, 4-sample chunk c) at c * (R * 16) + g * 128,
// so LBO = R * 16 and SBO = 128; row r, sample k sits at (k / 4) * R * 16 + r * 16 + (k % 4) * 4.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)(128 >> 4) << 32;
    return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

#define SD_D8(b) "+f"(d[(b) + 0]), "+f"(d[(b) + 1]), "+f"(d[(b) + 2]), "+f"(d[(b) + 3]), "+f"(d[(b) + 4]), "+f"(d[(b) + 5]), "+f"(d[(b) + 6]), "+f"(d[(b) + 7])

// D[64 x N] (+)= A[64 x 8] B[8 x N], TF32 operands K-major in shared memory, fp32 accumulators in registers
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "
        "%26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, "
        "%50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : SD_D8(0), SD_D8(8), SD_D8(16), SD_D8(24), SD_D8(32), SD_D8(40), SD_D8(48), SD_D8(56)
        : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "
        "%26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : SD_D8(0), SD_D8(8), SD_D8(16), SD_D8(24)
        : "l"(da), "l"(db), "r"(accumulate));
}
#undef SD_D8

struct TcArgs {
    int K, MI, NJ;
    float* C;
    long long ldc;
    float alpha, beta;
    int passes;          // 1 or 3
    int unbiased;        // round hi (slower, unbiased) instead of using the value the tensor core truncates
    const int2* tiles;   // (ti, tj) per tile
    int num_tiles;
    int a_strip;         // > 0: operand A is stored strip-major, [tile row][a_strip contraction rows][128 columns] (sd_cg.cu)
};

// Raw tile (TMA, [BK rows][32 columns] per box) -> K-major hi / lo copies.  Thread tt owns columns tt, tt + 128, ...: it reads
// one column of every box row (a warp reads 32 consecutive words) and writes 16-byte rows of core matrices (a warp writes 512
// consecutive bytes); both are free of bank conflicts.
template <int COLS>
__device__ __forceinline__ void transform_tile(uint32_t raw, uint32_t hi, uint32_t lo, int tt, bool split, bool unbiased)
{
#pragma unroll
    for (int c = tt; c < COLS; c += 128) {
        const uint32_t src = raw + (c / BOX_COLS) * BOX_BYTES + (c % BOX_COLS) * 4;
#pragma unroll
        for (int kc = 0; kc < BK / 4; ++kc) {
            float v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) v[u] = lds32(src + (kc * 4 + u) * (BOX_COLS * 4));
            const uint32_t off = kc * (COLS * 16) + c * 16;
            if (!split) {
                sts128(hi + off, make_float4(v[0], v[1], v[2], v[3]));
            } else if (unbiased) {
                float4 h, l;
                h.x = rna_tf32_bits(v[0]); h.y = rna_tf32_bits(v[1]); h.z = rna_tf32_bits(v[2]); h.w = rna_tf32_bits(v[3]);
                l.x = round_operand(v[0] - h.x); l.y = round_operand(v[1] - h.y);
                l.z = round_operand(v[2] - h.z); l.w = round_operand(v[3] - h.w);
                sts128(hi + off, h);
                sts128(lo + off, l);
            } else {
                // hi is the value as the tensor core sees it (low 13 mantissa bits ignored); the residual is rounded to TF32 so
                // that the hardware's truncation of the lo operand does not bias it
                float4 l;
                l.x = round_operand(v[0] - trunc_tf32(v[0])); l.y = round_operand(v[1] - trunc_tf32(v[1]));
                l.z = round_operand(v[2] - trunc_tf32(v[2])); l.w = round_operand(v[3] - trunc_tf32(v[3]));
                sts128(hi + off, make_float4(v[0], v[1], v[2], v[3]));
                sts128(lo + off, l);
            }
        }
    }
}

// =====================================================================================================
//   warp 0       TMA producer        (raw fp32 tiles of SA and SB, RAW_STAGES deep)
//   warps 4..7   transform           (raw -> K-major hi [and lo]; fence.proxy.async; KM_STAGES deep)
//   warps 8..15  two consumer warpgroups, 64 rows of C each: wgmma lo*hi, hi*lo, hi*hi per 8 samples, one fresh accumulator per
//                128-sample chunk folded into running sums in registers, then the write-back to C
// Register budget is rebalanced with setmaxnreg: the producer and transform warpgroups give registers back, the consumer
// warpgroups take them (chunk accumulator + running sums).
// =====================================================================================================
constexpr int T2_THREADS = 512;

template <int BN>
__global__ void __launch_bounds__(T2_THREADS, 1)
syrk_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const TcArgs a)
{
    using Cfg = TcCfg<BN>;
    constexpr int KM_STAGES = Cfg::KM_STAGES, NV = Cfg::NV;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned char* raw_base = smem;
    unsigned char* km_base = smem + RAW_STAGES * Cfg::RAW_BYTES;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::BAR_OFF);
    uint64_t* raw_full = bars;                                  // [RAW_STAGES] TMA bytes landed
    uint64_t* raw_empty = bars + RAW_STAGES;                    // [RAW_STAGES] transform has read the raw tile
    uint64_t* km_full = bars + 2 * RAW_STAGES;                  // [KM_STAGES] K-major operands written
    uint64_t* km_empty = bars + 2 * RAW_STAGES + KM_STAGES;     // [KM_STAGES] MMAs retired

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_k = (a.K + BK - 1) / BK;
    const bool split = a.passes == 3;

    if (threadIdx.x == 0) {
        for (int s = 0; s < RAW_STAGES; ++s) { mbar_init(&raw_full[s], 1); mbar_init(&raw_empty[s], 128); }
        for (int s = 0; s < KM_STAGES; ++s) { mbar_init(&km_full[s], 128); mbar_init(&km_empty[s], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
    }
    __syncthreads();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (warp == 0 && elect_one_sync()) {
            // ===================== TMA producer =====================
            uint32_t stage = 0, phase = 0;
            for (int t = blockIdx.x; t < a.num_tiles; t += gridDim.x) {
                const int2 tile = a.tiles[t];
                const int i0 = tile.x * BM, j0 = tile.y * BN;
                for (int kb = 0; kb < num_k; ++kb) {
                    mbar_wait(&raw_empty[stage], phase ^ 1);
                    mbar_arrive_expect_tx(&raw_full[stage], Cfg::RAW_BYTES);
                    unsigned char* sa = raw_base + stage * Cfg::RAW_BYTES;
                    unsigned char* sb = sa + RAW_A_BYTES;
                    const int k0 = kb * BK;
#pragma unroll
                    for (int cb = 0; cb < A_BLOCKS; ++cb)
                        tma_load_2d(sa + cb * BOX_BYTES, &map_a, &raw_full[stage], (a.a_strip ? 0 : i0) + cb * BOX_COLS, (a.a_strip ? tile.x * a.a_strip : 0) + k0);
#pragma unroll
                    for (int cb = 0; cb < Cfg::B_BLOCKS; ++cb) tma_load_2d(sb + cb * BOX_BYTES, &map_b, &raw_full[stage], j0 + cb * BOX_COLS, k0);
                    if (++stage == RAW_STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else if (warp < 8) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        // ===================== transform: raw -> K-major hi / lo =====================
        const int tt = threadIdx.x - 128;                 // 0..127
        uint32_t rs = 0, rph = 0, ks = 0, kph = 0;
        for (int t = blockIdx.x; t < a.num_tiles; t += gridDim.x) {
            for (int kb = 0; kb < num_k; ++kb) {
                mbar_wait(&raw_full[rs], rph);
                mbar_wait(&km_empty[ks], kph ^ 1);
                const uint32_t raw = smem_u32(raw_base + rs * Cfg::RAW_BYTES);
                const uint32_t hi = smem_u32(km_base + ks * Cfg::KM_BYTES);
                const uint32_t lo = hi + Cfg::KM_HALF;
                transform_tile<BM>(raw, hi, lo, tt, split, a.unbiased);
                transform_tile<BN>(raw + RAW_A_BYTES, hi + KM_A_BYTES, lo + KM_A_BYTES, tt, split, a.unbiased);
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
                mbar_arrive(&raw_empty[rs]);
                mbar_arrive(&km_full[ks]);
                if (++rs == RAW_STAGES) { rs = 0; rph ^= 1; }
                if (++ks == KM_STAGES) { ks = 0; kph ^= 1; }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 208;" ::: "memory");
        // ===================== consumers (warps 8..15) =====================
        const int wg = (warp - 8) >> 2;                   // 64-row half of the tile
        const int wq = warp & 3;                          // 16-row slice of the warpgroup
        const int g = lane >> 2, tq = lane & 3;
        const bool vec_ok = (a.ldc % 2 == 0) && ((reinterpret_cast<uintptr_t>(a.C) & 7) == 0);
        uint32_t ks = 0, kph = 0;
        int held = -1;                                    // stage whose MMAs may still be in flight
        float acc[NV];
        float run[NV];
        for (int t = blockIdx.x; t < a.num_tiles; t += gridDim.x) {
            const int2 tile = a.tiles[t];
#pragma unroll
            for (int v = 0; v < NV; ++v) { acc[v] = 0.f; run[v] = 0.f; }
            for (int kb = 0; kb < num_k; ++kb) {
                const bool chunk_first = (kb % KC_STAGES) == 0;
                const bool chunk_last = (kb % KC_STAGES) == KC_STAGES - 1 || kb == num_k - 1;
                mbar_wait(&km_full[ks], kph);
                const uint32_t a_hi = smem_u32(km_base + ks * Cfg::KM_BYTES) + wg * 64 * 16;
                const uint32_t b_hi = smem_u32(km_base + ks * Cfg::KM_BYTES) + KM_A_BYTES;
                const uint32_t a_lo = a_hi + Cfg::KM_HALF, b_lo = b_hi + Cfg::KM_HALF;
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < BK / 8; ++kk) {
                    const uint32_t oa = kk * 2 * (BM * 16), ob = kk * 2 * (BN * 16);     // two 4-sample chunks per k8 step
                    const uint32_t first = (chunk_first && kk == 0) ? 0u : 1u;
                    if (split) {
                        wgmma_tf32(acc, make_desc(a_lo + oa, BM * 16), make_desc(b_hi + ob, BN * 16), first);
                        wgmma_tf32(acc, make_desc(a_hi + oa, BM * 16), make_desc(b_lo + ob, BN * 16), 1u);
                        wgmma_tf32(acc, make_desc(a_hi + oa, BM * 16), make_desc(b_hi + ob, BN * 16), 1u);
                    } else {
                        wgmma_tf32(acc, make_desc(a_hi + oa, BM * 16), make_desc(b_hi + ob, BN * 16), first);
                    }
                }
                wgmma_commit();
                // One group stays in flight while the next stage is awaited: waiting for all but the newest group retires the
                // previous stage, whose shared memory goes back to the transform warps.  A chunk's last stage drains the
                // accumulator before it is folded.
                if (chunk_last) wgmma_wait0();
                else wgmma_wait1();
                __syncwarp();
                if (lane == 0) {
                    if (held >= 0) mbar_arrive(&km_empty[held]);
                    if (chunk_last) mbar_arrive(&km_empty[ks]);
                }
                held = chunk_last ? -1 : (int)ks;
                if (++ks == KM_STAGES) { ks = 0; kph ^= 1; }
                if (chunk_last) {
#pragma unroll
                    for (int v = 0; v < NV; ++v) run[v] = __fadd_rn(run[v], acc[v]);
                }
            }
            // write-back.  Accumulator fragment: register 4 j + 2 h + e holds row 16 wq + g + 8 h, column 8 j + 2 tq + e.
            // beta == 1 adds with fire-and-forget reductions (C is not read by the SM); every element is touched once per launch,
            // so the result is the single rounding of old + alpha * sum.
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int i = tile.x * BM + wg * 64 + wq * 16 + g + 8 * h;
                if (i >= a.MI) continue;
                float* crow = a.C + (long long)i * a.ldc;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const int c = tile.y * BN + 8 * j + 2 * tq;
                    if (c >= a.NJ) continue;
                    const float o0 = a.alpha * run[4 * j + 2 * h], o1 = a.alpha * run[4 * j + 2 * h + 1];
                    const bool two = c + 1 < a.NJ;
                    if (a.beta == 1.f) {
                        if (two && vec_ok)
                            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(crow + c), "f"(o0), "f"(o1) : "memory");
                        else {
                            atomicAdd(crow + c, o0);
                            if (two) atomicAdd(crow + c + 1, o1);
                        }
                    } else if (a.beta == 0.f) {
                        if (two && vec_ok) *reinterpret_cast<float2*>(crow + c) = make_float2(o0, o1);
                        else {
                            crow[c] = o0;
                            if (two) crow[c + 1] = o1;
                        }
                    } else {
                        crow[c] = fmaf(a.beta, crow[c], o0);
                        if (two) crow[c + 1] = fmaf(a.beta, crow[c + 1], o1);
                    }
                }
            }
        }
    }
}

int make_map(sd_ctx* ctx, CUtensorMap* map, const float* base, int64_t ld, int rows, int cols)
{
    sd_encode_tiled_fn enc = sd_encode_tiled();
    if (!enc) return sd_fail(ctx, SD_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
    cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)ld * sizeof(float)};
    cuuint32_t box[2] = {(cuuint32_t)BOX_COLS, (cuuint32_t)BK};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstride, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return sd_fail(ctx, SD_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
    return SD_OK;
}

}  // namespace

sd_encode_tiled_fn sd_encode_tiled()
{
    static sd_encode_tiled_fn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<sd_encode_tiled_fn>(p);
    }
    return fn;
}

bool sd_syrk_tc_supported(const float* d_S, int64_t lds, int K)
{
    // TMA needs a 16-byte aligned base and row pitch
    return K >= 1 && (reinterpret_cast<uintptr_t>(d_S) & 15) == 0 && (lds % 4) == 0;
}

// A prepared launch of the kernel: tensor maps, tile list (already on the device) and arguments.  Preparing costs two
// cuTensorMapEncodeTiled calls, the tile enumeration and a small host->device copy; iterative callers (sd_cg.cu) prepare once.
struct sd_tc_plan {
    CUtensorMap map_a, map_b;
    TcArgs args;
    int grid;
    int bn;              // kernel variant: columns of C per tile (128, or 64 for a narrow single tile column)
};
static_assert(sizeof(sd_tc_plan) <= SD_TC_PLAN_BYTES, "sd_tc_plan storage");

// C[i,j] = beta*C[i,j] + alpha * sum_{k<K} SA[k,i] * SB[k,j],  i < MI, j < NJ.   SA: K x MI (lda), SB: K x NJ (ldb), both row-major,
// i.e. both operands MN-major.  passes: 3 = 3xTF32 split (unbiased: hi rounded), 1 = one TF32 pass.  upper_only keeps the tiles
// that intersect j >= i (SYRK: SA == SB).  `rows` (optional) keeps the tiles whose C rows this rank owns (distributed trailing
// update).  C may alias SB when every CTA's column range of SB is read completely before its tile is written: true for MI <= 128
// (one tile row; each tile's operand columns are its own output columns).  d_tiles: device buffer for the tile list (at least
// sd_tc_max_tiles(MI, NJ) int2), or NULL to use the context's workspace.  *empty is set when no tile survives the filters
// (nothing to launch).
int sd_gemm_tn_tc_prepare(sd_ctx* ctx, const float* d_SA, int64_t lda, const float* d_SB, int64_t ldb, int K, int MI, int NJ,
                          float* d_C, int64_t ldc, float alpha, float beta, int passes, bool unbiased, bool upper_only,
                          const sd_row_filter* rows, void* d_tiles_buf, void* plan_storage, bool* empty, bool narrow, int a_strip_rows)
{
    sd_tc_plan* plan = reinterpret_cast<sd_tc_plan*>(plan_storage);
    *empty = true;
    if (MI <= 0 || NJ <= 0 || K <= 0) return SD_OK;
    SD_REQUIRE(ctx, passes == 1 || passes == 3, "passes must be 1 or 3");
    // operand A either as the row-major K x MI matrix, or strip-major: sd_div_up(MI, 128) strips of a_strip_rows x 128 floats each
    // (rows K .. a_strip_rows - 1 and the columns beyond MI hold zeros): a CTA then streams one contiguous strip
    SD_REQUIRE(ctx, a_strip_rows == 0 || (a_strip_rows % BK == 0 && a_strip_rows >= K), "strip-major operand: rows padded to the pipeline stage");
    int rc = a_strip_rows ? make_map(ctx, &plan->map_a, d_SA, BM, sd_div_up(MI, BM) * a_strip_rows, BM) : make_map(ctx, &plan->map_a, d_SA, lda, K, MI);
    if (rc) return rc;
    rc = make_map(ctx, &plan->map_b, d_SB, ldb, K, NJ);
    if (rc) return rc;

    // a single tile column of at most 64 columns runs the narrow variant
    const int BN = (narrow && NJ <= 64) ? 64 : 128;
    // tile list, ordered by super-tiles so that concurrently running tiles share operand columns in L2
    const int TI = sd_div_up(MI, BM), TJ = sd_div_up(NJ, BN);
    std::vector<int2>& tiles = ctx->tile_scratch;
    tiles.clear();
    for (int si = 0; si < TI; si += GI)
        for (int sj = 0; sj < TJ; sj += GJ)
            for (int ti = si; ti < si + GI && ti < TI; ++ti) {
                if (rows && rows->nranks > 1 && sd_panel_owner(rows->first_row + (int64_t)ti * BM, rows->nranks) != rows->rank) continue;
                for (int tj = sj; tj < sj + GJ && tj < TJ; ++tj)
                    if (!upper_only || tj * BN + BN - 1 >= ti * BM) tiles.push_back(make_int2(ti, tj));
            }
    if (tiles.empty()) return SD_OK;
    int2* d_tiles = (int2*)d_tiles_buf;
    if (!d_tiles) d_tiles = (int2*)sd_workspace(ctx, SD_WS_TC_TILES, tiles.size() * sizeof(int2));
    if (!d_tiles) return SD_ERR_CUDA;
    SD_CUDA(ctx, cudaMemcpyAsync(d_tiles, tiles.data(), tiles.size() * sizeof(int2), cudaMemcpyHostToDevice, ctx->stream));

    TcArgs& a = plan->args;
    a.K = K; a.MI = MI; a.NJ = NJ; a.C = d_C; a.ldc = ldc; a.alpha = alpha; a.beta = beta; a.passes = passes;
    a.unbiased = unbiased ? 1 : 0;
    a.a_strip = a_strip_rows;
    a.tiles = d_tiles; a.num_tiles = (int)tiles.size();
    const int sms = ctx->sm_count - ctx->syrk_sm_reserve > 0 ? ctx->sm_count - ctx->syrk_sm_reserve : 1;
    plan->grid = a.num_tiles < sms ? a.num_tiles : sms;
    plan->bn = BN;
    if (BN == 64) SD_CUDA(ctx, cudaFuncSetAttribute(syrk_wgmma_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<64>::SMEM_BYTES));
    else SD_CUDA(ctx, cudaFuncSetAttribute(syrk_wgmma_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<128>::SMEM_BYTES));
    *empty = false;
    return SD_OK;
}

int sd_gemm_tn_tc_launch(sd_ctx* ctx, const void* plan_storage)
{
    const sd_tc_plan* plan = reinterpret_cast<const sd_tc_plan*>(plan_storage);
    if (plan->bn == 64)
        syrk_wgmma_kernel<64><<<plan->grid, T2_THREADS, TcCfg<64>::SMEM_BYTES, ctx->stream>>>(plan->map_a, plan->map_b, plan->args);
    else
        syrk_wgmma_kernel<128><<<plan->grid, T2_THREADS, TcCfg<128>::SMEM_BYTES, ctx->stream>>>(plan->map_a, plan->map_b, plan->args);
    SD_LAUNCH_CHECK(ctx, "syrk_wgmma_kernel");
    return SD_OK;
}

int sd_syrk_tc(sd_ctx* ctx, const float* d_S, int64_t lds, int K, int MI, int NJ, float* d_C, int64_t ldc, float alpha, float beta,
               int passes, bool unbiased, const sd_row_filter* rows)
{
    alignas(64) unsigned char storage[SD_TC_PLAN_BYTES];
    bool empty = true;
    int rc = sd_gemm_tn_tc_prepare(ctx, d_S, lds, d_S, lds, K, MI, NJ, d_C, ldc, alpha, beta, passes, unbiased, true, rows,
                                   nullptr, storage, &empty, false, 0);
    if (rc || empty) return rc;
    return sd_gemm_tn_tc_launch(ctx, storage);
}
