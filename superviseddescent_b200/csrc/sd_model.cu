// rcr::detection_model on the device: load / save (cereal binary, byte compatible with the reference's
// face_landmarks_model_rcr_*.bin), align_mean, and the batched detect cascade.
//
//   file format    model.hpp:178-182 -> superviseddescent.hpp:356-360 -> regressors.hpp:395-399,164-168
//                  -> utils/mat_cerealisation.hpp:42-99 ; model.hpp:111-115 ; adaptive_vlhog.hpp:55-59
//   detect         model.hpp:132-157 -> superviseddescent.hpp:323-344 (predict: sequential over levels), on device frames or
//                  on host frames of any size, grey or colour, any number of faces each
#include "sd_internal.cuh"

#include <cuda.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <exception>
#include <fstream>
#include <string>
#include <vector>

struct sd_model {
    int device = 0;
    int num_levels = 0;
    int num_landmarks = 0;
    std::vector<int> rows, cols;
    std::vector<std::vector<float>> weights;      // host copies (for save / getters)
    std::vector<float*> d_weights;                // device copies
    std::vector<sd_regulariser> regs;
    std::vector<sd_hog_param> hog;
    std::vector<float> mean;
    float* d_mean = nullptr;                      // device copy of the mean (sd_track_faces aligns it on the device)
    std::vector<std::string> ids, right_ids, left_ids;
    sd_normalisation norm{};
};

namespace {

// ---- little-endian byte cursor over the whole file -------------------------------------------------
struct Cursor {
    const std::vector<unsigned char>& buf;
    size_t pos = 0;
    bool good = true;
    explicit Cursor(const std::vector<unsigned char>& b) : buf(b) {}
    template <class T> T get()
    {
        T v{};
        if (pos + sizeof(T) > buf.size()) { good = false; return v; }
        memcpy(&v, buf.data() + pos, sizeof(T));
        pos += sizeof(T);
        return v;
    }
    bool bytes(void* dst, size_t n)
    {
        if (pos + n > buf.size()) { good = false; return false; }
        memcpy(dst, buf.data() + pos, n);
        pos += n;
        return true;
    }
    std::vector<std::string> strings()
    {
        std::vector<std::string> out;
        const uint64_t n = get<uint64_t>();                 // cereal size_type
        if (!good || n > buf.size()) { good = false; return out; }
        for (uint64_t i = 0; i < n && good; ++i) {
            const uint64_t len = get<uint64_t>();
            if (!good || len > buf.size() - pos) { good = false; break; }
            out.emplace_back(reinterpret_cast<const char*>(buf.data() + pos), (size_t)len);
            pos += (size_t)len;
        }
        return out;
    }
    bool matrix(std::vector<float>& data, int& r, int& c)
    {
        r = get<int32_t>();
        c = get<int32_t>();
        const int32_t type = get<int32_t>();
        (void)get<uint8_t>();                               // isContinuous: same bytes either way for a packed Mat
        if (!good || type != 5 /* CV_32FC1 */ || r < 0 || c < 0) { good = false; return false; }
        if ((uint64_t)r * (uint64_t)c > (buf.size() - pos) / sizeof(float)) { good = false; return false; }   // corrupt header: do not allocate
        data.resize((size_t)r * c);
        return bytes(data.data(), data.size() * sizeof(float));
    }
};

struct Writer {
    std::vector<unsigned char> out;
    template <class T> void put(T v)
    {
        const unsigned char* p = reinterpret_cast<const unsigned char*>(&v);
        out.insert(out.end(), p, p + sizeof(T));
    }
    void strings(const std::vector<std::string>& v)
    {
        put<uint64_t>(v.size());
        for (const auto& s : v) { put<uint64_t>(s.size()); out.insert(out.end(), s.begin(), s.end()); }
    }
    void matrix(const std::vector<float>& d, int r, int c)
    {
        put<int32_t>(r); put<int32_t>(c); put<int32_t>(5); put<uint8_t>(1);
        const unsigned char* p = reinterpret_cast<const unsigned char*>(d.data());
        out.insert(out.end(), p, p + d.size() * sizeof(float));
    }
};

int resolve_eyes(sd_ctx* ctx, sd_model* m)
{
    auto find = [&](const std::string& s) {
        for (size_t i = 0; i < m->ids.size(); ++i) if (m->ids[i] == s) return (int)i;
        return -1;
    };
    if (m->right_ids.empty() || m->left_ids.empty() || m->right_ids.size() > SD_MAX_EYES || m->left_ids.size() > SD_MAX_EYES)
        return sd_fail(ctx, SD_ERR_INVALID, "a model needs 1..%d eye identifiers per eye", SD_MAX_EYES);
    m->norm.kind = 1;
    m->norm.n_right = (int)m->right_ids.size();
    m->norm.n_left = (int)m->left_ids.size();
    for (int i = 0; i < m->norm.n_right; ++i) {
        m->norm.right_idx[i] = find(m->right_ids[i]);
        if (m->norm.right_idx[i] < 0) return sd_fail(ctx, SD_ERR_MISSING_ID, "one of given rightEyeIdentifiers ids not present in lms");
    }
    for (int i = 0; i < m->norm.n_left; ++i) {
        m->norm.left_idx[i] = find(m->left_ids[i]);
        if (m->norm.left_idx[i] < 0) return sd_fail(ctx, SD_ERR_MISSING_ID, "one of given leftEyeIdentifiers ids not present in lms");
    }
    return SD_OK;
}

int validate_and_upload(sd_ctx* ctx, sd_model* m)
{
    const int L = m->num_landmarks;
    if (L < 1 || (int)m->mean.size() != 2 * L) return sd_fail(ctx, SD_ERR_INVALID, "mean must have 2L entries");
    for (int s = 0; s < m->num_levels; ++s) {
        const int D = sd_hog_feature_length(L, &m->hog[s]);
        if (m->rows[s] != D || m->cols[s] != 2 * L)
            return sd_fail(ctx, SD_ERR_INVALID, "level %d: regressor is %dx%d but the HOG parameters give %dx%d", s, m->rows[s], m->cols[s], D, 2 * L);
    }
    int rc = resolve_eyes(ctx, m);
    if (rc) return rc;
    m->device = ctx->device;
    m->d_weights.assign(m->num_levels, nullptr);
    SD_CUDA(ctx, cudaMalloc(&m->d_mean, m->mean.size() * sizeof(float)));
    SD_CUDA(ctx, cudaMemcpyAsync(m->d_mean, m->mean.data(), m->mean.size() * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    for (int s = 0; s < m->num_levels; ++s) {
        const size_t bytes = m->weights[s].size() * sizeof(float);
        SD_CUDA(ctx, cudaMalloc(&m->d_weights[s], bytes));
        SD_CUDA(ctx, cudaMemcpyAsync(m->d_weights[s], m->weights[s].data(), bytes, cudaMemcpyHostToDevice, ctx->stream));
    }
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SD_OK;
}

int detect_device(sd_ctx* ctx, const sd_model* m, const sd_image_batch* images, const int32_t* d_image_index, const float* d_x0,
                  int count, float* d_landmarks, uint8_t* d_face_degenerate = nullptr, const sd_sample_warp* d_warp = nullptr)
{
    const int L = m->num_landmarks, P = 2 * L;
    if (count <= 0) return SD_OK;
    // ping-pong landmark buffers
    float* xa = (float*)sd_workspace(ctx, SD_WS_SCRATCH, (size_t)2 * count * P * sizeof(float));
    if (!xa) return SD_ERR_CUDA;
    float* xb = xa + (size_t)count * P;
    SD_CUDA(ctx, cudaMemcpyAsync(xa, d_x0, (size_t)count * P * sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
    int maxD = 0;
    for (int s = 0; s < m->num_levels; ++s) maxD = m->rows[s] > maxD ? m->rows[s] : maxD;
    const int64_t ld = ((int64_t)maxD + 3) / 4 * 4;
    float* A = (float*)sd_workspace(ctx, SD_WS_FEATURES, (size_t)count * ld * sizeof(float));
    if (!A) return SD_ERR_CUDA;
    float* cur = xa;
    float* nxt = xb;
    for (int s = 0; s < m->num_levels; ++s) {               // superviseddescent.hpp:326-342
        int rc = sd_hog_batch_unmirrored(ctx, images, d_image_index, cur, P, count, L, &m->norm, &m->hog[s], A, ld, d_face_degenerate,
                                         d_warp);
        if (rc) return rc;
        rc = sd_cascade_update(ctx, A, ld, count, m->rows[s], m->d_weights[s], P, cur, &m->norm, nxt);
        if (rc) return rc;
        float* t = cur; cur = nxt; nxt = t;
    }
    SD_CUDA(ctx, cudaMemcpyAsync(d_landmarks, cur, (size_t)count * P * sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
    return SD_OK;
}


// ---- region-of-interest gather (sd_detect_faces_host, and sd_train_level / sd_apply_level on host frames) -------------------
// The cascade only ever reads a neighbourhood of the face, so instead of copying whole frames over PCIe a small kernel pulls
// the ROI rows of every face straight out of the caller's PINNED host frame (zero-copy loads through the unified address
// space, 16-byte vectors) into a packed grey device buffer.  In detect, if a patch later needs a frame pixel outside its ROI
// the HOG kernel raises d_roi_miss[face] and that face is repeated from its full frame, so the result never depends on the
// ROI heuristic; a training level plans its regions exactly (sd_train.cu).

// 16 interleaved B,G,R pixels (48 bytes) -> 16 grey bytes
__device__ __forceinline__ uint4 bgr16_to_gray(const uint4 (&v)[3])
{
    const uint32_t w[12] = {v[0].x, v[0].y, v[0].z, v[0].w, v[1].x, v[1].y, v[1].z, v[1].w, v[2].x, v[2].y, v[2].z, v[2].w};
    uint32_t out[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        uint32_t o = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int b = 3 * (4 * q + k);                  // byte index of the pixel's B (little endian words)
            o |= sd_bgr_to_gray((w[b >> 2] >> (8 * (b & 3))) & 255u, (w[(b + 1) >> 2] >> (8 * ((b + 1) & 3))) & 255u,
                                (w[(b + 2) >> 2] >> (8 * ((b + 2) & 3))) & 255u) << (8 * k);
        }
        out[q] = o;
    }
    return make_uint4(out[0], out[1], out[2], out[3]);
}

// C = channels of the source frames.  One step moves 16 pixels: one uint4 of grey, or three of B,G,R (the ROI's x is a
// multiple of 16 pixels, so 48 k bytes into a 16-byte aligned row) converted on the way.
template <int C>
__global__ void __launch_bounds__(256) roi_gather_kernel(const GatherRec* __restrict__ rec, int n, uint8_t* __restrict__ dst)
{
    constexpr int U = 4;                                    // steps in flight per thread before the stores: PCIe read latency is ~1 us
    for (int f = blockIdx.x; f < n; f += gridDim.x) {
        const GatherRec r = rec[f];
        const int total = r.vec_per_row * r.rows;
        uint8_t* d = dst + r.dst_offset;
        for (int i0 = threadIdx.x; i0 < total; i0 += U * blockDim.x) {
            uint4 v[U][C];
            int row[U], col[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int i = i0 + u * blockDim.x;
                row[u] = i / r.vec_per_row;
                col[u] = i - row[u] * r.vec_per_row;
                if (i < total) {
                    const uint4* s = reinterpret_cast<const uint4*>(r.src + (long long)row[u] * r.src_stride) + C * col[u];
#pragma unroll
                    for (int c = 0; c < C; ++c) v[u][c] = s[c];
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (i0 + u * blockDim.x >= total) continue;
                uint4 g;
                if constexpr (C == 1) g = v[u][0];
                else g = bgr16_to_gray(v[u]);
                reinterpret_cast<uint4*>(d + (long long)row[u] * 16 * r.vec_per_row)[col[u]] = g;
            }
        }
    }
}

// conservative ROI of one face: landmark bounding box of the initialisation, grown by the largest patch half size of the
// schedule plus a drift allowance, clipped to the frame, x aligned to 16 pixels; row_pixels = pixels a row of the caller's
// buffer holds (row_stride / channels), which the ROI never reaches past
sd_roi face_roi(const sd_model* m, const float* x0, int width, int height, int row_pixels)
{
    const int L = m->num_landmarks;
    float minx = x0[0], maxx = x0[0], miny = x0[L], maxy = x0[L];
    for (int i = 1; i < L; ++i) {
        minx = x0[i] < minx ? x0[i] : minx; maxx = x0[i] > maxx ? x0[i] : maxx;
        miny = x0[i + L] < miny ? x0[i + L] : miny; maxy = x0[i + L] > maxy ? x0[i + L] : maxy;
    }
    float rxs = 0, rys = 0, lxs = 0, lys = 0;
    for (int i = 0; i < m->norm.n_right; ++i) { rxs += x0[m->norm.right_idx[i]]; rys += x0[m->norm.right_idx[i] + L]; }
    for (int i = 0; i < m->norm.n_left; ++i) { lxs += x0[m->norm.left_idx[i]]; lys += x0[m->norm.left_idx[i] + L]; }
    rxs /= m->norm.n_right; rys /= m->norm.n_right; lxs /= m->norm.n_left; lys /= m->norm.n_left;
    const float ied = std::sqrt((rxs - lxs) * (rxs - lxs) + (rys - lys) * (rys - lys));
    // per level: half patch (the IED may grow a little) + how far the landmarks may have drifted by then (none at level 0)
    float grow = 0.f;
    for (size_t l = 0; l < m->hog.size(); ++l) {
        const float g = 0.5f * m->hog[l].relative_patch_size * ied * 1.1f + (l > 0 ? 0.2f * ied : 0.f);
        grow = g > grow ? g : grow;
    }
    grow += 4.f;
    int xa = (int)std::floor(minx - grow), xb = (int)std::ceil(maxx + grow);
    int ya = (int)std::floor(miny - grow), yb = (int)std::ceil(maxy + grow);
    xa = xa < 0 ? 0 : xa; ya = ya < 0 ? 0 : ya;
    xb = xb > width ? width : xb; yb = yb > height ? height : yb;
    sd_roi r{};
    if (xb <= xa || yb <= ya) { xa = 0; ya = 0; xb = 16 < width ? 16 : width; yb = 1; }   // face entirely outside the frame
    r.x = xa & ~15;
    int w = ((xb - r.x) + 15) & ~15;
    const int maxw = (row_pixels - r.x) & ~15;
    if (w > maxw) w = maxw;
    r.w = w; r.y = ya; r.h = yb - ya; r.row_stride = w; r.reserved = 0; r.offset = 0;
    return r;
}

typedef CUresult (*PFN_pointerGetAttribute)(void* data, CUpointer_attribute attribute, CUdeviceptr ptr);

}  // namespace

int sd_roi_gather(sd_ctx* ctx, const GatherRec* d_grey, int n_grey, const GatherRec* d_colour, int n_colour, uint8_t* dst, cudaStream_t stream)
{
    const int most = 8 * ctx->sm_count;
    if (n_grey > 0) {
        roi_gather_kernel<1><<<n_grey < most ? n_grey : most, 256, 0, stream>>>(d_grey, n_grey, dst);
        SD_LAUNCH_CHECK(ctx, "roi_gather_kernel<1>");
    }
    if (n_colour > 0) {
        roi_gather_kernel<3><<<n_colour < most ? n_colour : most, 256, 0, stream>>>(d_colour, n_colour, dst);
        SD_LAUNCH_CHECK(ctx, "roi_gather_kernel<3>");
    }
    return SD_OK;
}

// Frames inside the last pinned allocation seen (every frame of sd_detect_batch_host's batch) are mapped by offset.
const uint8_t* sd_mapped_frame(const uint8_t* p, size_t bytes, PinnedRange& last)
{
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    if (a >= last.lo && a + bytes <= last.hi) return reinterpret_cast<const uint8_t*>(a + last.delta);
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    if (attr.type != cudaMemoryTypeHost || !attr.devicePointer) return nullptr;
    static PFN_pointerGetAttribute get = nullptr;
    if (!get) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuPointerGetAttribute", &fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            get = reinterpret_cast<PFN_pointerGetAttribute>(fn);
    }
    CUdeviceptr start = 0;
    size_t size = 0;
    if (get && get(&start, CU_POINTER_ATTRIBUTE_RANGE_START_ADDR, (CUdeviceptr)a) == CUDA_SUCCESS &&
        get(&size, CU_POINTER_ATTRIBUTE_RANGE_SIZE, (CUdeviceptr)a) == CUDA_SUCCESS && start <= a && a + bytes <= start + size) {
        last.lo = start; last.hi = start + size;
        last.delta = (intptr_t)reinterpret_cast<uintptr_t>(attr.devicePointer) - (intptr_t)a;
    }
    return static_cast<const uint8_t*>(attr.devicePointer);
}

int sd_check_host_frame(sd_ctx* ctx, const char* fn, const sd_host_frame& fr, int f)
{
    if (fr.channels != 1 && fr.channels != 3)
        return sd_fail(ctx, SD_ERR_INVALID, "%s: frame %d has %d channels (1 or 3)", fn, f, fr.channels);
    if (!fr.h_data || fr.width <= 0 || fr.height <= 0 || (int64_t)fr.row_stride < (int64_t)fr.width * fr.channels)
        return sd_fail(ctx, SD_ERR_INVALID, "%s: frame %d: bad data pointer, size or row_stride < width * channels", fn, f);
    return SD_OK;
}

int sd_ensure_stage(sd_ctx* ctx, size_t bytes)
{
    for (int b = 0; b < 2; ++b) {
        if (ctx->stage_bytes[b] < bytes) {
            if (ctx->d_stage[b]) { SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); SD_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream)); SD_CUDA(ctx, cudaFree(ctx->d_stage[b])); ctx->d_stage[b] = nullptr; }
            SD_CUDA(ctx, cudaMalloc(&ctx->d_stage[b], bytes));
            ctx->stage_bytes[b] = bytes;
        }
    }
    return SD_OK;
}

namespace {

size_t bgr_bytes(const sd_host_frame& f) { return f.channels == 3 ? (size_t)f.height * sd_round16(3 * (size_t)f.width) : 0; }

// ---- host frames -> grey device frames (sd_detect_faces_host's chunks, sd_upload_frames), laid out by sd_gray_layout -----
// Copies frames[0..n) to the layout desc describes at d_gray, on the copy stream once free_ev (recorded on the compute stream:
// nothing still reads the destination or d_bgr) has completed.  Grey frames go straight to their place; colour frames go as
// B,G,R rows at a 16-byte pitch, back to back from d_bgr (bgr_bytes each), and the compute stream converts them into place
// (sd_bgr2gray) after ready_ev, which marks the end of the copies.
int upload_frames(sd_ctx* ctx, const sd_host_frame* frames, const sd_frame* desc, int n, uint8_t* d_gray, uint8_t* d_bgr,
                  cudaEvent_t free_ev, cudaEvent_t ready_ev)
{
    SD_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, free_ev, 0));
    uint8_t* bgr = d_bgr;
    for (int i = 0; i < n; ++i) {
        const sd_host_frame& f = frames[i];
        uint8_t* dst = f.channels == 3 ? bgr : d_gray + desc[i].offset;
        const size_t pitch = f.channels == 3 ? sd_round16(3 * (size_t)f.width) : (size_t)desc[i].row_stride;
        if ((size_t)f.row_stride == pitch)
            SD_CUDA(ctx, cudaMemcpyAsync(dst, f.h_data, sd_host_frame_bytes(f), cudaMemcpyHostToDevice, ctx->copy_stream));
        else
            SD_CUDA(ctx, cudaMemcpy2DAsync(dst, pitch, f.h_data, f.row_stride, (size_t)f.width * f.channels, f.height,
                                           cudaMemcpyHostToDevice, ctx->copy_stream));
        bgr += bgr_bytes(f);
    }
    SD_CUDA(ctx, cudaEventRecord(ready_ev, ctx->copy_stream));
    SD_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ready_ev, 0));
    bgr = d_bgr;
    for (int i = 0; i < n; ++i) {
        const sd_host_frame& f = frames[i];
        if (f.channels != 3) continue;
        const int rc = sd_bgr2gray(ctx, bgr, f.width, f.height, (int64_t)sd_round16(3 * (size_t)f.width), 0, 1, d_gray + desc[i].offset,
                                   desc[i].row_stride, 0);
        if (rc) return rc;
        bgr += bgr_bytes(f);
    }
    return SD_OK;
}

// Full route: faces grouped by frame, every referenced frame copied to the device once (upload_frames; a chunk's B,G,R bytes
// behind its grey frames), chunks double-buffered against the cascade.  x0 / out: count x 2L in the caller's face order.
int detect_faces_full(sd_ctx* ctx, const sd_model* m, const sd_host_frame* frames, const int32_t* face_frame, int count,
                      const float* x0, float* out)
{
    const int P = 2 * m->num_landmarks;
    const size_t chunk_cap = (size_t)128 << 20;              // frame bytes per staging buffer (at least one frame)
    std::vector<int> order(count);
    for (int i = 0; i < count; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return face_frame[a] < face_frame[b]; });
    std::vector<int> up;                                      // referenced frames in upload order
    std::vector<int32_t> local(count);                        // per sorted face: its frame's index in `up`, then in its chunk
    for (int k = 0; k < count; ++k) {
        if (up.empty() || up.back() != face_frame[order[k]]) up.push_back(face_frame[order[k]]);
        local[k] = (int32_t)up.size() - 1;
    }
    std::vector<sd_host_frame> fr(up.size());
    for (size_t u = 0; u < up.size(); ++u) fr[u] = frames[up[u]];
    std::vector<int> chunk_first;                             // first upload of each chunk
    size_t used = 0, need = 0;
    for (size_t u = 0; u < fr.size(); ++u) {
        const size_t b = sd_gray_bytes(fr[u]) + bgr_bytes(fr[u]);
        if (chunk_first.empty() || used + b > chunk_cap) { chunk_first.push_back((int)u); used = 0; }
        used += b;
        need = used > need ? used : need;
    }
    chunk_first.push_back((int)fr.size());
    // per chunk: the grey layout of its frames in its staging buffer (descriptor offsets from the buffer), B,G,R bytes after it
    const int nc = (int)chunk_first.size() - 1;
    std::vector<sd_frame> desc(fr.size());
    std::vector<size_t> bgr_at(nc);
    std::vector<char> uniform(nc);
    for (int c = 0; c < nc; ++c) {
        bool same = true;
        bgr_at[c] = sd_gray_layout(fr.data() + chunk_first[c], chunk_first[c + 1] - chunk_first[c], desc.data() + chunk_first[c], &same);
        uniform[c] = same;
    }
    std::vector<int> face_first(chunk_first.size(), count);   // first sorted face of each chunk
    std::vector<int> chunk_of(up.size());
    for (size_t c = 0; c + 1 < chunk_first.size(); ++c)
        for (int u = chunk_first[c]; u < chunk_first[c + 1]; ++u) chunk_of[u] = (int)c;
    for (int k = count - 1; k >= 0; --k) {                    // faces of a chunk are contiguous in sorted order
        const int c = chunk_of[local[k]];
        face_first[c] = k;
        local[k] -= chunk_first[c];                           // frame index inside its chunk
    }
    int rc = sd_ensure_stage(ctx, need);
    if (rc) return rc;
    // device tables: landmarks (in, out) in sorted order, face -> frame index, frame descriptors
    std::vector<float> xs((size_t)count * P);
    for (int k = 0; k < count; ++k) memcpy(&xs[(size_t)k * P], x0 + (size_t)order[k] * P, P * sizeof(float));
    const size_t xbytes = (size_t)count * P * sizeof(float);
    const size_t ibytes = sd_round16((size_t)count * sizeof(int32_t));
    unsigned char* tab = (unsigned char*)sd_workspace(ctx, SD_WS_PARTIAL, 2 * xbytes + ibytes + up.size() * sizeof(sd_frame));
    if (!tab) return SD_ERR_CUDA;
    float* d_x = (float*)tab;
    float* d_out = (float*)(tab + xbytes);
    int32_t* d_idx = (int32_t*)(tab + 2 * xbytes);
    sd_frame* d_desc = (sd_frame*)(tab + 2 * xbytes + ibytes);
    SD_CUDA(ctx, cudaMemcpyAsync(d_x, xs.data(), xbytes, cudaMemcpyHostToDevice, ctx->stream));
    SD_CUDA(ctx, cudaMemcpyAsync(d_idx, local.data(), (size_t)count * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    SD_CUDA(ctx, cudaMemcpyAsync(d_desc, desc.data(), desc.size() * sizeof(sd_frame), cudaMemcpyHostToDevice, ctx->stream));
    // the copy stream must not run ahead of work already queued on the compute stream that still reads the staging buffers
    SD_CUDA(ctx, cudaEventRecord(ctx->stage_done[0], ctx->stream));
    SD_CUDA(ctx, cudaEventRecord(ctx->stage_done[1], ctx->stream));
    int buf = 0;
    for (int c = 0; c < nc; ++c, buf ^= 1) {
        const int u0 = chunk_first[c], u1 = chunk_first[c + 1];
        uint8_t* stage = (uint8_t*)ctx->d_stage[buf];
        rc = upload_frames(ctx, fr.data() + u0, desc.data() + u0, u1 - u0, stage, stage + bgr_at[c], ctx->stage_done[buf], ctx->stage_ev[buf]);
        if (rc) return rc;
        const sd_image_batch ib = sd_gray_batch(stage, desc.data() + u0, u1 - u0, uniform[c], d_desc + u0);
        const int k0 = face_first[c], n = face_first[c + 1] - k0;
        rc = detect_device(ctx, m, &ib, d_idx + k0, d_x + (size_t)k0 * P, n, d_out + (size_t)k0 * P);
        if (rc) return rc;
        SD_CUDA(ctx, cudaEventRecord(ctx->stage_done[buf], ctx->stream));
    }
    SD_CUDA(ctx, cudaMemcpyAsync(xs.data(), d_out, xbytes, cudaMemcpyDeviceToHost, ctx->stream));
    rc = sd_check_hog_status(ctx, "detect");                  // synchronises
    if (rc) return rc;
    for (int k = 0; k < count; ++k) memcpy(out + (size_t)order[k] * P, &xs[(size_t)k * P], P * sizeof(float));
    return SD_OK;
}

// ROI route: every referenced frame is pinned and device-mapped (mapped[f]), with 16-byte aligned base and rows
int detect_faces_roi(sd_ctx* ctx, const sd_model* m, const sd_host_frame* frames, const std::vector<const uint8_t*>& mapped,
                     const int32_t* face_frame, int count, const float* x0, float* out)
{
    const int P = 2 * m->num_landmarks;
    const size_t chunk_cap = SD_STAGE_HALF_BYTES;             // packed grey ROI bytes per staging buffer
    // the ROI of every face, from its own frame's size; faces are grouped into chunks that fit one staging buffer
    std::vector<sd_roi> rois(count);
    std::vector<sd_frame> dims(count);
    std::vector<int> chunk_first;
    size_t used = 0;
    for (int i = 0; i < count; ++i) {
        const sd_host_frame& f = frames[face_frame[i]];
        sd_roi r = face_roi(m, x0 + (size_t)i * P, f.width, f.height, f.row_stride / f.channels);
        const size_t bytes = (size_t)r.row_stride * r.h;
        if (bytes > chunk_cap)                                // a face window larger than a staging buffer: whole-frame route
            return detect_faces_full(ctx, m, frames, face_frame, count, x0, out);
        if (chunk_first.empty() || used + bytes > chunk_cap) { chunk_first.push_back(i); used = 0; }
        r.offset = (int64_t)used;
        used += bytes;
        rois[i] = r;
        dims[i] = sd_frame{f.width, f.height, 0, 0, 0};      // with d_roi only the frame size is read
    }
    chunk_first.push_back(count);
    // gather records per chunk: grey faces first, then colour faces (one launch each)
    std::vector<GatherRec> recs(count);
    std::vector<int> chunk_grey(chunk_first.size(), 0);
    for (size_t c = 0; c + 1 < chunk_first.size(); ++c) {
        int k = chunk_first[c];
        for (int ch = 1; ch <= 3; ch += 2)
            for (int i = chunk_first[c]; i < chunk_first[c + 1]; ++i) {
                const sd_host_frame& f = frames[face_frame[i]];
                if (f.channels != ch) continue;
                const sd_roi& r = rois[i];
                recs[k++] = GatherRec{mapped[face_frame[i]] + (int64_t)r.y * f.row_stride + (int64_t)r.x * ch, f.row_stride, r.offset,
                                      r.w >> 4, r.h};
                if (ch == 1) ++chunk_grey[c];
            }
    }
    int rc = sd_ensure_stage(ctx, chunk_cap + (1u << 20));
    if (rc) return rc;
    // device tables: landmarks (in, out), ROI records, frame sizes, gather records, miss flags
    const size_t xbytes = (size_t)count * P * sizeof(float);
    const size_t rbytes = (size_t)count * sizeof(sd_roi);
    const size_t fbytes = (size_t)count * sizeof(sd_frame);
    const size_t gbytes = (size_t)count * sizeof(GatherRec);
    unsigned char* tab = (unsigned char*)sd_workspace(ctx, SD_WS_PARTIAL, 2 * xbytes + rbytes + fbytes + gbytes + count + 64);
    if (!tab) return SD_ERR_CUDA;
    float* d_x = (float*)tab;
    float* d_out = (float*)(tab + xbytes);
    sd_roi* d_roi = (sd_roi*)(tab + 2 * xbytes);
    sd_frame* d_dims = (sd_frame*)(tab + 2 * xbytes + rbytes);
    GatherRec* d_rec = (GatherRec*)(tab + 2 * xbytes + rbytes + fbytes);
    uint8_t* d_miss = tab + 2 * xbytes + rbytes + fbytes + gbytes;
    SD_CUDA(ctx, cudaMemcpyAsync(d_x, x0, xbytes, cudaMemcpyHostToDevice, ctx->stream));
    SD_CUDA(ctx, cudaMemcpyAsync(d_roi, rois.data(), rbytes, cudaMemcpyHostToDevice, ctx->stream));
    SD_CUDA(ctx, cudaMemcpyAsync(d_dims, dims.data(), fbytes, cudaMemcpyHostToDevice, ctx->stream));
    SD_CUDA(ctx, cudaMemcpyAsync(d_rec, recs.data(), gbytes, cudaMemcpyHostToDevice, ctx->stream));
    SD_CUDA(ctx, cudaMemsetAsync(d_miss, 0, count, ctx->stream));
    SD_CUDA(ctx, cudaEventRecord(ctx->stage_done[0], ctx->stream));
    SD_CUDA(ctx, cudaEventRecord(ctx->stage_done[1], ctx->stream));
    int buf = 0;
    for (size_t c = 0; c + 1 < chunk_first.size(); ++c, buf ^= 1) {
        const int first = chunk_first[c], n = chunk_first[c + 1] - first, ng = chunk_grey[c];
        SD_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->stage_done[buf], 0));   // also orders the table uploads before the first gather
        // the SMs read the chunk's ROI rows zero-copy from the pinned frames: no host cores are spent packing rows at link speed
        rc = sd_roi_gather(ctx, d_rec + first, ng, d_rec + first + ng, n - ng, (uint8_t*)ctx->d_stage[buf], ctx->copy_stream);
        if (rc) return rc;
        SD_CUDA(ctx, cudaEventRecord(ctx->stage_ev[buf], ctx->copy_stream));
        SD_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->stage_ev[buf], 0));
        sd_image_batch ib{};
        ib.d_data = (const uint8_t*)ctx->d_stage[buf];
        ib.count = n;
        ib.d_roi = d_roi + first;
        ib.d_roi_miss = d_miss + first;
        ib.d_frames = d_dims + first;
        rc = detect_device(ctx, m, &ib, nullptr, d_x + (size_t)first * P, n, d_out + (size_t)first * P);
        if (rc) return rc;
        SD_CUDA(ctx, cudaEventRecord(ctx->stage_done[buf], ctx->stream));
    }
    std::vector<uint8_t> miss(count);
    SD_CUDA(ctx, cudaMemcpyAsync(out, d_out, xbytes, cudaMemcpyDeviceToHost, ctx->stream));
    SD_CUDA(ctx, cudaMemcpyAsync(miss.data(), d_miss, count, cudaMemcpyDeviceToHost, ctx->stream));
    rc = sd_check_hog_status(ctx, "detect");                  // synchronises
    if (rc) return rc;
    // faces whose cascade wandered outside the gathered region: repeat them from their full frames
    std::vector<int> again;
    for (int i = 0; i < count; ++i) if (miss[i]) again.push_back(i);
    if (again.empty()) return SD_OK;
    ctx->roi_fallbacks += (int64_t)again.size();
    const int na = (int)again.size();
    std::vector<int32_t> ff(na);
    std::vector<float> xa((size_t)na * P), xo((size_t)na * P);
    for (int j = 0; j < na; ++j) {
        ff[j] = face_frame[again[j]];
        memcpy(&xa[(size_t)j * P], x0 + (size_t)again[j] * P, P * sizeof(float));
    }
    rc = detect_faces_full(ctx, m, frames, ff.data(), na, xa.data(), xo.data());
    if (rc) return rc;
    for (int j = 0; j < na; ++j) memcpy(out + (size_t)again[j] * P, &xo[(size_t)j * P], P * sizeof(float));
    return SD_OK;
}

}  // namespace

namespace {
// apps/rcr/rcr-train.cpp:149-212: one warp per row; cv::norm's float differences / double sum / double sqrt, the result
// stored as float (:169) and multiplied by the float factor (float)(1.0f / IED(prediction)).
__global__ void landmark_error_kernel(const float* __restrict__ pred, long long ldp, const float* __restrict__ gt, long long ldgt, int N,
                                      int L, const sd_eyes_dev eyes, float* __restrict__ err, long long lde)
{
    const int r = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= N) return;
    const float* p = pred + (long long)r * ldp;
    const float* g = gt + (long long)r * ldgt;
    const double ied = sd_device_ied(p, L, eyes);
    const float f = (float)(1.0 / ied);
    for (int i = lane; i < L; i += 32) {
        const float dx = __fsub_rn(p[i], g[i]), dy = __fsub_rn(p[i + L], g[i + L]);
        const float n = (float)sqrt(__dadd_rn(__dmul_rn((double)dx, (double)dx), __dmul_rn((double)dy, (double)dy)));
        err[(long long)r * lde + i] = __fmul_rn(n, f);
    }
}
}  // namespace

extern "C" {

int sd_align_mean(const float* h_mean, int L, int box_x, int box_y, int box_w, int box_h, float sx, float sy,
                  float tx, float ty, float* h_out)
{
    if (!h_mean || !h_out || L < 1) return SD_ERR_INVALID;
    // model.hpp:72-73.  OpenCV folds (m*s + 0.5f + t) * w + x into one scaled conversion
    // m * (float)(s*w) + (float)((0.5 + t)*w + x), evaluated in float (mul, then add).
    const float ax = (float)((double)sx * (double)box_w);
    const float bx = (float)(((double)0.5f + (double)tx) * (double)box_w + (double)box_x);
    const float ay = (float)((double)sy * (double)box_h);
    const float by = (float)(((double)0.5f + (double)ty) * (double)box_h + (double)box_y);
    for (int i = 0; i < L; ++i) {
        volatile float px = h_mean[i] * ax;        // volatile: keep mul and add un-fused on any host compiler
        h_out[i] = px + bx;
        volatile float py = h_mean[i + L] * ay;
        h_out[i + L] = py + by;
    }
    return SD_OK;
}

int sd_perturb_box(int box_x, int box_y, int box_w, int box_h, float tx, float ty, float scaling, int32_t out_box[4])
{
    if (!out_box) return SD_ERR_INVALID;
    // rcr-train.cpp:133-143, float arithmetic; volatile keeps every product / sum a separately rounded float
    volatile float tx_pixel = tx * (float)box_w;
    volatile float ty_pixel = ty * (float)box_h;
    volatile float pw = (float)box_w * scaling;
    volatile float ph = (float)box_h * scaling;
    volatile float hx = ((float)box_w - pw) / 2.0f, hy = ((float)box_h - ph) / 2.0f;
    volatile float x = (float)box_x + hx, y = (float)box_y + hy;
    out_box[0] = (int32_t)(x + tx_pixel);
    out_box[1] = (int32_t)(y + ty_pixel);
    out_box[2] = (int32_t)pw;
    out_box[3] = (int32_t)ph;
    return SD_OK;
}

int sd_normalised_landmark_errors(sd_ctx* ctx, const float* d_pred, int64_t ldp, const float* d_gt, int64_t ldgt, int N, int L,
                                  const sd_normalisation* eyes, float* d_err, int64_t lde)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, d_pred && d_gt && d_err && N >= 0 && L >= 1 && ldp >= 2 * L && ldgt >= 2 * L && lde >= L, "bad argument");
    SD_REQUIRE(ctx, eyes && eyes->kind == 1, "the normalised error needs the eye landmark indices");
    if (N == 0) return SD_OK;
    sd_eyes_dev eyes_dev;
    int rc = sd_eyes_to_dev(ctx, eyes, L, &eyes_dev);
    if (rc) return rc;
    landmark_error_kernel<<<sd_div_up(N, 4), 128, 0, ctx->stream>>>(d_pred, ldp, d_gt, ldgt, N, L, eyes_dev, d_err, lde);
    SD_LAUNCH_CHECK(ctx, "landmark_error_kernel");
    return SD_OK;
}

static int model_load_impl(sd_ctx* ctx, const char* path, sd_model** out)
{
    std::ifstream f(path, std::ios::binary);
    if (!f) return sd_fail(ctx, SD_ERR_IO, "The given model file could not be opened: %s", path);   // model.hpp:199
    std::vector<unsigned char> buf((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    Cursor c(buf);
    sd_model* m = new sd_model();
    auto bail = [&](const char* why) { delete m; return sd_fail(ctx, SD_ERR_IO, "%s: %s", why, path); };

    const uint64_t nreg = c.get<uint64_t>();                 // vector<LinearRegressor>
    if (!c.good || nreg == 0 || nreg > 256) return bail("not a detection_model archive (regressor count)");
    m->num_levels = (int)nreg;
    m->rows.resize(nreg); m->cols.resize(nreg); m->weights.resize(nreg); m->regs.resize(nreg);
    for (uint64_t i = 0; i < nreg; ++i) {
        if (!c.matrix(m->weights[i], m->rows[i], m->cols[i])) return bail("truncated regressor matrix");
        m->regs[i].type = c.get<int32_t>();                  // Regulariser: type, lambda, regularise_last_row
        m->regs[i].param = c.get<float>();
        m->regs[i].regularise_last_row = c.get<uint8_t>();
    }
    const auto n_ids = c.strings();                          // InterEyeDistanceNormalisation's own copies
    const auto n_right = c.strings();
    const auto n_left = c.strings();
    int mr = 0, mc = 0;
    if (!c.matrix(m->mean, mr, mc)) return bail("truncated mean");
    m->ids = c.strings();
    const uint64_t nhog = c.get<uint64_t>();
    if (!c.good || nhog != nreg) return bail("hog_params count differs from the regressor count");
    m->hog.resize(nhog);
    for (uint64_t i = 0; i < nhog; ++i) {
        m->hog[i].variant = c.get<int32_t>();
        m->hog[i].num_cells = c.get<int32_t>();
        m->hog[i].cell_size = c.get<int32_t>();
        m->hog[i].num_bins = c.get<int32_t>();
        m->hog[i].relative_patch_size = c.get<float>();
    }
    m->right_ids = c.strings();
    m->left_ids = c.strings();
    if (!c.good || c.pos != buf.size()) return bail("truncated archive or trailing bytes");
    if (mr != 1 || n_ids != m->ids || n_right != m->right_ids || n_left != m->left_ids)
        return bail("inconsistent archive (normaliser ids differ from the model's)");
    m->num_landmarks = (int)m->ids.size();
    int rc = validate_and_upload(ctx, m);
    if (rc) { sd_model_destroy(m); return rc; }
    *out = m;
    return SD_OK;
}

int sd_model_load(sd_ctx* ctx, const char* path, sd_model** out)
{
    if (!ctx || !path || !out) return SD_ERR_INVALID;
    *out = nullptr;
    try {                                                     // nothing may unwind through the C boundary
        return model_load_impl(ctx, path, out);
    } catch (const std::exception& e) {
        return sd_fail(ctx, SD_ERR_IO, "could not read %s: %s", path, e.what());
    } catch (...) {
        return sd_fail(ctx, SD_ERR_IO, "could not read %s", path);
    }
}

int sd_model_save(sd_ctx* ctx, const sd_model* m, const char* path)
{
    if (!ctx || !m || !path) return SD_ERR_INVALID;
    Writer w;
    w.put<uint64_t>((uint64_t)m->num_levels);
    for (int i = 0; i < m->num_levels; ++i) {
        w.matrix(m->weights[i], m->rows[i], m->cols[i]);
        w.put<int32_t>(m->regs[i].type);
        w.put<float>(m->regs[i].param);
        w.put<uint8_t>(m->regs[i].regularise_last_row ? 1 : 0);
    }
    w.strings(m->ids); w.strings(m->right_ids); w.strings(m->left_ids);
    w.matrix(m->mean, 1, 2 * m->num_landmarks);
    w.strings(m->ids);
    w.put<uint64_t>((uint64_t)m->num_levels);
    for (int i = 0; i < m->num_levels; ++i) {
        w.put<int32_t>(m->hog[i].variant); w.put<int32_t>(m->hog[i].num_cells); w.put<int32_t>(m->hog[i].cell_size);
        w.put<int32_t>(m->hog[i].num_bins); w.put<float>(m->hog[i].relative_patch_size);
    }
    w.strings(m->right_ids); w.strings(m->left_ids);
    std::ofstream f(path, std::ios::binary);
    if (!f) return sd_fail(ctx, SD_ERR_IO, "could not open %s for writing", path);
    f.write(reinterpret_cast<const char*>(w.out.data()), (std::streamsize)w.out.size());
    return f.good() ? SD_OK : sd_fail(ctx, SD_ERR_IO, "short write to %s", path);
}

int sd_model_create(sd_ctx* ctx, int num_levels, int num_landmarks, const float* const* h_weights,
                    const sd_regulariser* regs, const sd_hog_param* hog_params, const float* h_mean,
                    const char* const* landmark_ids, const char* const* right_eye_ids, int n_right,
                    const char* const* left_eye_ids, int n_left, sd_model** out)
{
    if (!ctx || !out) return SD_ERR_INVALID;
    *out = nullptr;
    SD_REQUIRE(ctx, num_levels >= 1 && num_landmarks >= 1 && h_weights && regs && hog_params && h_mean && landmark_ids &&
                        right_eye_ids && left_eye_ids, "null / empty argument");
    sd_model* m = new sd_model();
    m->num_levels = num_levels;
    m->num_landmarks = num_landmarks;
    for (int i = 0; i < num_landmarks; ++i) m->ids.emplace_back(landmark_ids[i]);
    for (int i = 0; i < n_right; ++i) m->right_ids.emplace_back(right_eye_ids[i]);
    for (int i = 0; i < n_left; ++i) m->left_ids.emplace_back(left_eye_ids[i]);
    m->mean.assign(h_mean, h_mean + 2 * num_landmarks);
    m->rows.resize(num_levels); m->cols.resize(num_levels); m->weights.resize(num_levels);
    m->regs.assign(regs, regs + num_levels);
    m->hog.assign(hog_params, hog_params + num_levels);
    for (int s = 0; s < num_levels; ++s) {
        m->rows[s] = sd_hog_feature_length(num_landmarks, &hog_params[s]);
        m->cols[s] = 2 * num_landmarks;
        m->weights[s].assign(h_weights[s], h_weights[s] + (size_t)m->rows[s] * m->cols[s]);
    }
    int rc = validate_and_upload(ctx, m);
    if (rc) { sd_model_destroy(m); return rc; }
    *out = m;
    return SD_OK;
}

void sd_model_destroy(sd_model* m)
{
    if (!m) return;
    cudaSetDevice(m->device);
    for (float* p : m->d_weights) if (p) cudaFree(p);
    if (m->d_mean) cudaFree(m->d_mean);
    delete m;
}

int sd_model_num_levels(const sd_model* m) { return m ? m->num_levels : -1; }
int sd_model_num_landmarks(const sd_model* m) { return m ? m->num_landmarks : -1; }
int sd_model_hog_param(const sd_model* m, int level, sd_hog_param* out)
{
    if (!m || !out || level < 0 || level >= m->num_levels) return SD_ERR_INVALID;
    *out = m->hog[level];
    return SD_OK;
}
int sd_model_regulariser(const sd_model* m, int level, sd_regulariser* out)
{
    if (!m || !out || level < 0 || level >= m->num_levels) return SD_ERR_INVALID;
    *out = m->regs[level];
    return SD_OK;
}
int sd_model_normalisation(const sd_model* m, sd_normalisation* out)
{
    if (!m || !out) return SD_ERR_INVALID;
    *out = m->norm;
    return SD_OK;
}
int sd_model_get_mean(const sd_model* m, float* h_mean)
{
    if (!m || !h_mean) return SD_ERR_INVALID;
    memcpy(h_mean, m->mean.data(), m->mean.size() * sizeof(float));
    return SD_OK;
}
int sd_model_get_weights(const sd_model* m, int level, float* h_w, int* rows, int* cols)
{
    if (!m || level < 0 || level >= m->num_levels) return SD_ERR_INVALID;
    if (rows) *rows = m->rows[level];
    if (cols) *cols = m->cols[level];
    if (h_w) memcpy(h_w, m->weights[level].data(), m->weights[level].size() * sizeof(float));
    return SD_OK;
}
const char* sd_model_landmark_id(const sd_model* m, int i)
{
    if (!m || i < 0 || i >= m->num_landmarks) return nullptr;
    return m->ids[i].c_str();
}

int sd_detect_batch_device(sd_ctx* ctx, const sd_model* m, const sd_image_batch* images, const float* d_x0, int count,
                           float* d_landmarks)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, m && images && d_x0 && d_landmarks && count >= 0, "bad argument");
    SD_REQUIRE(ctx, images->count >= count, "fewer images than faces");
    const int rc = detect_device(ctx, m, images, nullptr, d_x0, count, d_landmarks);
    if (rc) return rc;
    // a degenerate face (inter-eye distance too small for a patch) or a bad frame index is an error here, as it is in the
    // reference (cv::resize on an empty ROI throws); reading the flag synchronises the stream
    return sd_check_hog_status(ctx, "detect");
}

int sd_detect_faces_device(sd_ctx* ctx, const sd_model* m, const sd_image_batch* images, const int32_t* d_face_frame,
                           const float* d_x0, int num_faces, float* d_landmarks)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, m && images && d_x0 && d_landmarks && num_faces >= 0, "bad argument");
    if (!d_face_frame) SD_REQUIRE(ctx, images->count >= num_faces, "fewer images than faces");
    const int rc = detect_device(ctx, m, images, d_face_frame, d_x0, num_faces, d_landmarks);
    if (rc) return rc;
    return sd_check_hog_status(ctx, "detect");                // also reports a face index out of range
}

int sd_detect_faces_device_warped(sd_ctx* ctx, const sd_model* m, const sd_image_batch* images, const int32_t* d_face_frame,
                                  const sd_sample_warp* d_warp, const float* d_x0, int num_faces, float* d_landmarks)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, m && images && d_warp && d_x0 && d_landmarks && num_faces >= 0, "bad argument");
    SD_REQUIRE(ctx, !images->d_roi, "a warped batch must hold whole frames (no d_roi)");
    if (!d_face_frame) SD_REQUIRE(ctx, images->count >= num_faces, "fewer images than faces");
    const int rc = detect_device(ctx, m, images, d_face_frame, d_x0, num_faces, d_landmarks, nullptr, d_warp);
    if (rc) return rc;
    return sd_check_hog_status(ctx, "detect");                // also reports a face index out of range or an invalid warp
}

int sd_detect_faces_host(sd_ctx* ctx, const sd_model* m, const sd_host_frame* frames, int num_frames, const int32_t* h_face_frame,
                         int num_faces, const int32_t* h_boxes, const float* h_x0, float* h_landmarks)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, m && num_frames >= 0 && num_faces >= 0, "bad argument");
    if (num_faces == 0) return SD_OK;
    SD_REQUIRE(ctx, frames && h_face_frame && h_landmarks, "null argument");
    SD_REQUIRE(ctx, (h_boxes == nullptr) != (h_x0 == nullptr), "exactly one of h_boxes and h_x0 must be given");
    std::vector<char> used(num_frames, 0);
    for (int i = 0; i < num_faces; ++i) {
        if (h_face_frame[i] < 0 || h_face_frame[i] >= num_frames)
            return sd_fail(ctx, SD_ERR_INVALID, "%s: face %d refers to frame %d of %d", __func__, i, h_face_frame[i], num_frames);
        used[h_face_frame[i]] = 1;
    }
    for (int f = 0; f < num_frames; ++f) {
        const int rc = used[f] ? sd_check_host_frame(ctx, __func__, frames[f], f) : SD_OK;
        if (rc) return rc;
    }
    const int L = m->num_landmarks, P = 2 * L;
    // initial landmarks: align_mean of each box on the host (model.hpp:135), or the caller's
    std::vector<float> x0;
    if (h_boxes) {
        x0.resize((size_t)num_faces * P);
        for (int i = 0; i < num_faces; ++i)
            sd_align_mean(m->mean.data(), L, h_boxes[4 * i], h_boxes[4 * i + 1], h_boxes[4 * i + 2], h_boxes[4 * i + 3], 1.f, 1.f, 0.f, 0.f,
                          &x0[(size_t)i * P]);
    }
    const float* xs = h_boxes ? x0.data() : h_x0;
    // ROI route when every referenced frame is in pinned, device-mapped host memory with 16-byte aligned rows
    std::vector<const uint8_t*> mapped(num_frames, nullptr);
    PinnedRange last;
    bool roi = true;
    for (int f = 0; f < num_frames && roi; ++f) {
        if (!used[f]) continue;
        mapped[f] = sd_mapped_frame(frames[f].h_data, sd_host_frame_bytes(frames[f]), last);
        roi = mapped[f] && ((reinterpret_cast<uintptr_t>(mapped[f]) | (uintptr_t)frames[f].row_stride) & 15) == 0;
    }
    if (roi) return detect_faces_roi(ctx, m, frames, mapped, h_face_frame, num_faces, xs, h_landmarks);
    return detect_faces_full(ctx, m, frames, h_face_frame, num_faces, xs, h_landmarks);
}

int sd_detect_batch_host(sd_ctx* ctx, const sd_model* m, const uint8_t* h_images, int count, int width, int height,
                         int row_stride, const int32_t* h_boxes, float* h_landmarks)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, m && h_images && h_boxes && h_landmarks && count >= 0 && width > 0 && height > 0 && row_stride >= width, "bad argument");
    // frame i at h_images + i * height * row_stride, face i in frame i
    std::vector<sd_host_frame> frames(count);
    std::vector<int32_t> face_frame(count);
    for (int i = 0; i < count; ++i) {
        frames[i] = sd_host_frame{h_images + (size_t)i * height * row_stride, width, height, row_stride, 1};
        face_frame[i] = i;
    }
    return sd_detect_faces_host(ctx, m, frames.data(), count, face_frame.data(), count, h_boxes, nullptr, h_landmarks);
}

int sd_upload_frames(sd_ctx* ctx, const sd_host_frame* frames, int count, void* d_buf, size_t* bytes, sd_image_batch* out)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, frames && count >= 1 && bytes, "bad argument");
    for (int f = 0; f < count; ++f) {
        const int rc = sd_check_host_frame(ctx, __func__, frames[f], f);
        if (rc) return rc;
    }
    std::vector<sd_frame> desc(count);
    bool uniform = true;
    const size_t gray = sd_gray_layout(frames, count, desc.data(), &uniform);
    const size_t need = gray + (uniform ? 0 : (size_t)count * sizeof(sd_frame));   // the descriptors follow the grey frames
    if (!d_buf) { *bytes = need; return SD_OK; }
    SD_REQUIRE(ctx, out && (reinterpret_cast<uintptr_t>(d_buf) & 15) == 0 && *bytes >= need,
               "d_buf must be 16-byte aligned and hold the size the query gives; out must not be NULL");
    uint8_t* base = static_cast<uint8_t*>(d_buf);
    // Colour frames pass through the B,G,R scratch about 64 MB at a time, so the scratch stays small when a training set is
    // uploaded.  The staging events are free: sd_detect_faces_host records them anew before it waits on them, and this call
    // returns only when its own work is done.
    const size_t chunk_cap = (size_t)64 << 20;
    for (int i0 = 0, i1; i0 < count; i0 = i1) {
        size_t b = bgr_bytes(frames[i0]);
        for (i1 = i0 + 1; i1 < count && b + bgr_bytes(frames[i1]) <= chunk_cap; ++i1) b += bgr_bytes(frames[i1]);
        uint8_t* bgr = (uint8_t*)sd_workspace(ctx, SD_WS_UPLOAD, b);
        if (!bgr) return SD_ERR_CUDA;
        SD_CUDA(ctx, cudaEventRecord(ctx->stage_done[0], ctx->stream));
        const int rc = upload_frames(ctx, frames + i0, desc.data() + i0, i1 - i0, base, bgr, ctx->stage_done[0], ctx->stage_ev[0]);
        if (rc) return rc;
    }
    if (!uniform)
        SD_CUDA(ctx, cudaMemcpyAsync(base + gray, desc.data(), (size_t)count * sizeof(sd_frame), cudaMemcpyHostToDevice, ctx->stream));
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));        // the caller may free or reuse the host frames
    *out = sd_gray_batch(base, desc.data(), count, uniform, reinterpret_cast<const sd_frame*>(base + gray));
    return SD_OK;
}

}  // extern "C"

int sd_detect_device(sd_ctx* ctx, const sd_model* m, const sd_image_batch* images, const int32_t* d_face_frame, const float* d_x0,
                     int count, float* d_landmarks, uint8_t* d_face_degenerate, const sd_sample_warp* d_warp)
{
    return detect_device(ctx, m, images, d_face_frame, d_x0, count, d_landmarks, d_face_degenerate, d_warp);
}

const float* sd_model_device_mean(const sd_model* m) { return m->d_mean; }
