// ColPivHouseholderQRSolver's diagnostic (regressors.hpp:288-293): numerical rank of the regularised A^T A.
//
// The reference runs Eigen::ColPivHouseholderQR on the D x D matrix only to ask rank() / isInvertible() and to print
// "The regularised AtA is not invertible ... (The rank is r, full rank would be D). Increase lambda."; the weights then come
// from the explicit inverse.  A^T A + Lambda is symmetric positive SEMI-definite, and for that class the rank-revealing
// factorisation is the diagonally pivoted Cholesky (LAPACK xPSTRF): at step k the largest remaining Schur-complement diagonal
// d_k is the pivot (ties: the smallest index), and rank = #{k : d_k > threshold * d_0} with Eigen's default threshold eps * D;
// the factorisation stops at the first pivot at or below it (or <= 0).
//
// No row or column swaps: a chosen index is marked dead and its later factor entries are 0.  Blocked right-looking, in panels
// of kRankNb pivots, on a working copy C of the upper triangle (the solve still needs G):
//   panel   one persistent kernel over all SMs runs the panel's pivots in sequence.  Per pivot every CTA reduces the per-CTA
//           arg-max candidates of the live diagonal (the same answer on every CTA: max with smallest-index ties is a total order),
//           forms its slice of column p of the current Schur complement, C[:,p] - sum_{m<k} Lt[m][:] Lt[m][p], scales it into
//           row k of the panel Lt, downdates the live diagonal and posts its next candidate; one grid barrier per pivot.
//   update  C -= Lt^T Lt over the whole matrix (dead rows included: they are never read again) on the SYRK dispatcher
//           (syrk_upper, the Cholesky's trailing update): about D^3 flops in all.
//   stop    the host reads the accepted pivot count and the stop flag after every panel (one synchronise per panel).
// Every sum has a fixed order and the SYRK touches each element once per launch, so the rank is reproducible bit for bit.
#include "sd_internal.cuh"

#include <cstring>

namespace {

constexpr int kRankNb = 128;          // pivots per panel
constexpr int kRankThreads = 512;

struct RankState {
    int rank;                          // pivots accepted so far
    int stop;                          // 1: a pivot fell to the threshold, or every index is taken
    float d0, dlast;                   // first and last accepted pivot
    unsigned int barrier;              // arrivals at the grid barrier of the running panel
};

struct PanelArgs {
    const float* C;                    // working copy, upper triangle, pitch ldc
    float* Lt;                         // kRankNb x ldc: row k = factor column of the panel's k-th pivot
    float* dwork;                      // live diagonal; -1: chosen
    float2* best;                      // [2][gridDim.x] per-CTA candidates (value, index bits), double-buffered by pivot parity
    RankState* st;
    long long ldc;
    int D, k0, npiv;                   // global index of the panel's first pivot; pivots this panel may take
    float threshold;
};

__device__ __forceinline__ bool better(float v, int i, float bv, int bi)
{
    return v > bv || (v == bv && i >= 0 && (bi < 0 || i < bi));
}

// arg-max (largest value, smallest index on ties) over the block; every thread gets the result
__device__ void block_argmax(float& v, int& i, float* red_v, int* red_i)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (better(ov, oi, v, i)) { v = ov; i = oi; }
    }
    __syncthreads();                                                  // red_* may still be read from the previous call
    if (lane == 0) { red_v[warp] = v; red_i[warp] = i; }
    __syncthreads();
    v = lane < kRankThreads / 32 ? red_v[lane] : -1.f;
    i = lane < kRankThreads / 32 ? red_i[lane] : -1;
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (better(ov, oi, v, i)) { v = ov; i = oi; }
    }
}

// grid barrier of a cooperative launch: arrivals are counted in st->barrier (zeroed before the launch); bounded, a protocol
// bug must trap (context error), never hang the GPU
__device__ __forceinline__ void grid_barrier(unsigned int* count, unsigned int target)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(count, 1u);
        const long long t0 = clock64();
        while (*reinterpret_cast<volatile unsigned int*>(count) < target) {
            if (clock64() - t0 > 8000000000LL) __trap();
        }
        __threadfence();
    }
    __syncthreads();
}

__global__ void rank_diag_init_kernel(const float* __restrict__ C, long long ldc, int D, float* __restrict__ dwork)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < D) dwork[i] = C[(long long)i * ldc + i];
}

__global__ void __launch_bounds__(kRankThreads, 1) rank_panel_kernel(const PanelArgs a)
{
    __shared__ float red_v[kRankThreads / 32];
    __shared__ int red_i[kRankThreads / 32];
    __shared__ float s_lp[kRankNb];                                   // Lt[m][p] of the panel's earlier pivots
    const int tid = threadIdx.x, cta = blockIdx.x, grid = gridDim.x;
    const long long stride = (long long)grid * kRankThreads;
    const long long first = (long long)cta * kRankThreads + tid;
    unsigned int arrivals = 0;
    // this CTA's candidate from the live diagonal as the previous panel's update left it
    float bv = -1.f;
    int bi = -1;
    for (long long i = first; i < a.D; i += stride) {
        const float v = a.dwork[i];
        if (better(v, (int)i, bv, bi)) { bv = v; bi = (int)i; }
    }
    block_argmax(bv, bi, red_v, red_i);
    if (tid == 0) a.best[cta] = make_float2(bv, __int_as_float(bi));
    arrivals += grid;
    grid_barrier(&a.st->barrier, arrivals);
    float d0 = __ldcg(&a.st->d0), dlast = __ldcg(&a.st->dlast);
    int k = 0;
    for (; k < a.npiv; ++k) {
        // the pivot: every CTA reduces all candidates to the same answer.  Data other CTAs wrote during this launch (candidates,
        // factor entries) is read through L2 (__ldcg): the SM's L1 is not coherent with their stores.
        const float2* cand = a.best + (k & 1) * grid;
        float pv = -1.f;
        int p = -1;
        for (int c = tid; c < grid; c += kRankThreads) {
            const float2 e = __ldcg(cand + c);
            if (better(e.x, __float_as_int(e.y), pv, p)) { pv = e.x; p = __float_as_int(e.y); }
        }
        block_argmax(pv, p, red_v, red_i);
        if (a.k0 + k == 0) d0 = pv;
        if (p < 0 || !(pv > a.threshold * d0) || !(pv > 0.f)) break;   // numerically zero from here on
        dlast = pv;
        const float r = sqrtf(pv);
        const float inv_r = 1.0f / r;
        if (tid < k) s_lp[tid] = __ldcg(a.Lt + (long long)tid * a.ldc + p);
        __syncthreads();
        float* Lk = a.Lt + (long long)k * a.ldc;
        bv = -1.f;
        bi = -1;
        for (long long i = first; i < a.D; i += stride) {
            float acc = (i <= p) ? a.C[i * a.ldc + p] : a.C[(long long)p * a.ldc + i];   // symmetric: the upper triangle is stored
            const float* col = a.Lt + i;
#pragma unroll 8
            for (int m = 0; m < k; ++m) acc = fmaf(-col[(long long)m * a.ldc], s_lp[m], acc);
            const float di = a.dwork[i];
            float l = 0.f, nd = di;
            if (i == p) { l = r; nd = -1.f; }
            else if (di >= 0.f) { l = acc * inv_r; nd = di - l * l; nd = nd > 0.f ? nd : 0.f; }
            Lk[i] = l;
            a.dwork[i] = nd;
            if (better(nd, (int)i, bv, bi)) { bv = nd; bi = (int)i; }
        }
        block_argmax(bv, bi, red_v, red_i);
        if (tid == 0) a.best[((k + 1) & 1) * grid + cta] = make_float2(bv, __int_as_float(bi));
        arrivals += grid;
        grid_barrier(&a.st->barrier, arrivals);
    }
    if (cta == 0 && tid == 0) {
        a.st->rank = a.k0 + k;
        a.st->stop = (k < a.npiv || a.k0 + k == a.D) ? 1 : 0;
        a.st->d0 = d0;
        a.st->dlast = dlast;
    }
}

}  // namespace

// rank of the symmetric matrix whose upper triangle is in G (D x D, pitch ldg)
int sd_gram_rank(sd_ctx* ctx, const float* d_G, int64_t ldg, int D, int* rank_out, float* first_pivot, float* last_pivot)
{
    *rank_out = -1;
    const int64_t ldc = ((int64_t)D + 3) / 4 * 4;
    int grid = sd_div_up(D, kRankThreads);
    int per_sm = 0;
    SD_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rank_panel_kernel, kRankThreads, 0));
    if (per_sm < 1) return sd_fail(ctx, SD_ERR_CUDA, "sd_gram_rank: the panel kernel does not fit an SM");
    if (grid > ctx->sm_count) grid = ctx->sm_count;
    // [C: D x ldc][Lt: kRankNb x ldc][dwork: ldc][best: 2 x grid float2][state]
    const size_t n_c = (size_t)D * ldc, n_l = (size_t)kRankNb * ldc;
    const size_t bytes = (n_c + n_l + ldc + 4 * (size_t)grid) * sizeof(float) + sizeof(RankState);
    float* ws = (float*)sd_workspace(ctx, SD_WS_RANK, bytes);
    if (!ws) return SD_ERR_CUDA;
    float* C = ws;
    float* Lt = C + n_c;
    float* dwork = Lt + n_l;
    float2* best = reinterpret_cast<float2*>(dwork + ldc);
    RankState* st = reinterpret_cast<RankState*>(best + 2 * grid);
    SD_CUDA(ctx, cudaMemcpy2DAsync(C, ldc * sizeof(float), d_G, ldg * sizeof(float), (size_t)D * sizeof(float), D, cudaMemcpyDeviceToDevice, ctx->stream));
    SD_CUDA(ctx, cudaMemsetAsync(Lt, 0, n_l * sizeof(float), ctx->stream));
    SD_CUDA(ctx, cudaMemsetAsync(st, 0, sizeof(RankState), ctx->stream));
    rank_diag_init_kernel<<<sd_div_up(D, 256), 256, 0, ctx->stream>>>(C, ldc, D, dwork);
    SD_LAUNCH_CHECK(ctx, "rank_diag_init_kernel");
    PanelArgs args;
    args.C = C; args.Lt = Lt; args.dwork = dwork; args.best = best; args.st = st; args.ldc = ldc; args.D = D;
    args.threshold = 1.1920929e-7f * (float)D;                        // Eigen: NumTraits<float>::epsilon() * diagonalSize
    RankState* h = reinterpret_cast<RankState*>(reinterpret_cast<char*>(ctx->h_scratch) + 128);
    for (int k0 = 0;;) {
        args.k0 = k0;
        args.npiv = D - k0 < kRankNb ? D - k0 : kRankNb;
        SD_CUDA(ctx, cudaMemsetAsync(&st->barrier, 0, sizeof(unsigned int), ctx->stream));
        void* params[] = {&args};
        SD_CUDA(ctx, cudaLaunchCooperativeKernel((const void*)rank_panel_kernel, dim3(grid), dim3(kRankThreads), params, 0, ctx->stream));
        SD_LAUNCH_CHECK(ctx, "rank_panel_kernel");
        SD_CUDA(ctx, cudaMemcpyAsync(h, st, sizeof(RankState), cudaMemcpyDeviceToHost, ctx->stream));
        SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        const int kp = h->rank - k0;
        if (h->stop) break;
        int rc = syrk_upper(ctx, Lt, ldc, kp, D, D, C, ldc, -1.0f, 1.0f, syrk_is_big(kp, D, D), /*unbiased=*/true);
        if (rc) return rc;
        k0 = h->rank;
    }
    *rank_out = h->rank;
    if (first_pivot) *first_pivot = h->d0;
    if (last_pivot) *last_pivot = h->dlast;
    return SD_OK;
}
