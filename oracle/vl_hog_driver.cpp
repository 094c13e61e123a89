// TEST INFRASTRUCTURE ONLY.  One program written against the hog.h API alone (VLFeat's VlHog object), compiled twice: against
// the reference's hog.h + hog.c (oracle/vl_hog_api_ref.py builds oracle/_ref/vl_hog_driver_ref) and against this project's
// drop-in superviseddescent_b200/include/rcr/hog.h with libsd_b200 (tests/test_gpu_hog_h.py).  Both builds run the same fixed
// case list on the same seeded inputs and dump every result, so the test compares them record by record.
//
//   vl_hog_driver OUT [threads]
//
// Inputs come from vl_hog_driver_value (an integer LCG step per element, restated in tests/test_gpu_hog_h.py).  Records, in
// case order: int32 n, int32 ints[n], int64 m, float data[m].  ints = tag (1 put, 2 render), the case's parameters, then for a
// put hogW, hogH, dd, glyph size and the permutation; data = the extracted features, or the rendered image.  After every put
// the host input is overwritten before extract, so a put that had not finished reading it shows.  With "threads", four threads
// run the cases, each case on its own objects, and the records are written in the same order.
extern "C" {
#include "rcr/hog.h"
}

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <functional>
#include <string>
#include <thread>
#include <vector>

namespace {

struct Record {
    std::vector<int32_t> ints;
    std::vector<float> data;
};

float vl_hog_driver_value(uint64_t seed, uint64_t i)
{
    uint64_t x = seed * 0x9E3779B97F4A7C15ull + i;
    x = x * 6364136223846793005ull + 1442695040888963407ull;
    return (float)(x >> 40) * (1.0f / 16777216.0f);     // [0, 1), 24 bits
}

std::vector<float> values(uint64_t seed, size_t n, float scale, float shift)
{
    std::vector<float> v(n);
    for (size_t i = 0; i < n; ++i) v[i] = vl_hog_driver_value(seed, i) * scale + shift;
    return v;
}

Record extracted(VlHog* hog, std::vector<int32_t> params, std::vector<float>& input)
{
    for (float& v : input) v = 12345.f;                  // the caller may reuse its buffer as soon as the put returns
    Record r;
    r.ints = params;
    const int w = (int)vl_hog_get_width(hog), h = (int)vl_hog_get_height(hog), dd = (int)vl_hog_get_dimension(hog);
    r.ints.insert(r.ints.end(), {w, h, dd, (int)vl_hog_get_glyph_size(hog)});
    const vl_index* perm = vl_hog_get_permutation(hog);
    for (int d = 0; d < dd; ++d) r.ints.push_back((int32_t)perm[d]);
    r.data.resize((size_t)w * h * dd);
    vl_hog_extract(hog, r.data.data());
    return r;
}

// put_image: W x H buffer of C channels (values in [0, 255)), seed = case index
Record put_image(VlHog* hog, int seed, int W, int H, int C, int cs, int K, int variant, int bil, int tr)
{
    std::vector<float> img = values((uint64_t)seed, (size_t)W * H * C, 255.f, 0.f);
    vl_hog_put_image(hog, img.data(), W, H, C, cs);
    return extracted(hog, {1, 0, seed, W, H, C, cs, K, variant, bil, tr, 0}, img);
}

Record one_put_image(int seed, int W, int H, int C, int cs, int K, int variant, int bil, int tr)
{
    VlHog* hog = vl_hog_new(variant ? VlHogVariantUoctti : VlHogVariantDalalTriggs, K, tr);
    vl_hog_set_use_bilinear_orientation_assignments(hog, bil);
    Record r = put_image(hog, seed, W, H, C, cs, K, variant, bil, tr);
    vl_hog_delete(hog);
    return r;
}

// put_polar_field: modulus in [-0.5, 3.5) (a negative one does not vote), angle in [-10, 10) radians
Record one_put_polar(int seed, int W, int H, int cs, int K, int variant, int bil, int tr, int directed)
{
    VlHog* hog = vl_hog_new(variant ? VlHogVariantUoctti : VlHogVariantDalalTriggs, K, tr);
    vl_hog_set_use_bilinear_orientation_assignments(hog, bil);
    std::vector<float> mod = values((uint64_t)seed, (size_t)W * H, 4.f, -0.5f);
    std::vector<float> ang = values((uint64_t)seed + 1000, (size_t)W * H, 20.f, -10.f);
    vl_hog_put_polar_field(hog, mod.data(), ang.data(), directed, W, H, cs);
    Record r = extracted(hog, {1, 1, seed, W, H, 1, cs, K, variant, bil, tr, directed}, mod);
    vl_hog_delete(hog);
    return r;
}

// render of w x h cells of features into an image that starts non-zero, with one NaN pixel: random signed features (source 0),
// or the features of a put_image of a (w * cs) x (h * cs) image (source 1)
Record one_render(int seed, int w, int h, int K, int variant, int tr, int source)
{
    VlHog* hog = vl_hog_new(variant ? VlHogVariantUoctti : VlHogVariantDalalTriggs, K, tr);
    const int dd = (int)vl_hog_get_dimension(hog), g = (int)vl_hog_get_glyph_size(hog);
    std::vector<float> feat;
    if (source == 0) {
        feat = values((uint64_t)seed, (size_t)dd * w * h, 2.f, -1.f);
    } else {
        const int cs = 8;
        std::vector<float> img = values((uint64_t)seed, (size_t)w * cs * h * cs, 255.f, 0.f);
        vl_hog_put_image(hog, img.data(), w * cs, h * cs, 1, cs);
        feat.resize((size_t)dd * w * h);
        vl_hog_extract(hog, feat.data());
    }
    Record r;
    r.ints = {2, source, seed, w, h, K, variant, tr};
    r.data = values((uint64_t)seed + 2000, (size_t)w * g * h * g, 0.5f, -0.25f);
    r.data[r.data.size() / 3] = NAN;
    vl_hog_render(hog, r.data.data(), feat.data(), w, h);
    vl_hog_delete(hog);
    return r;
}

}  // namespace

int main(int argc, char** argv)
{
    if (argc < 2) {
        std::fprintf(stderr, "usage: %s OUT [threads]\n", argv[0]);
        return 2;
    }
    std::vector<std::function<std::vector<Record>()>> cases;
    int seed = 0;
    // put_image: W, H, channels, cell size, K, variant, bilinear, transposed
    const int images[][8] = {
        {4, 4, 1, 1, 1, 1, 0, 0},        {4, 4, 1, 4, 4, 0, 0, 1},         {5, 7, 3, 1, 16, 1, 1, 1},
        {37, 29, 3, 4, 9, 1, 1, 0},      {37, 29, 3, 4, 9, 1, 1, 1},       {55, 55, 1, 11, 4, 1, 0, 0},
        {55, 55, 1, 11, 4, 0, 1, 1},     {64, 48, 16, 8, 16, 1, 0, 1},     {64, 48, 16, 8, 16, 0, 1, 0},
        {120, 97, 1, 32, 9, 1, 0, 0},    {97, 120, 3, 32, 1, 0, 1, 1},     {160, 120, 1, 8, 9, 1, 0, 1},
        {640, 480, 3, 8, 9, 1, 1, 0},    {640, 480, 1, 4, 4, 0, 0, 1},     {1280, 720, 16, 11, 16, 0, 0, 0},
        {1920, 1080, 1, 8, 9, 1, 0, 0},  {1920, 1080, 3, 8, 9, 1, 1, 1},
    };
    for (const auto& c : images) {
        const int s = seed++;
        cases.push_back([=] { return std::vector<Record>{one_put_image(s, c[0], c[1], c[2], c[3], c[4], c[5], c[6], c[7])}; });
    }
    // one object reused across sizes (hog.c reallocates its buffers when the cell grid changes), either orientation
    for (int tr = 0; tr < 2; ++tr) {
        const int s = seed;
        seed += 4;
        cases.push_back([=] {
            VlHog* hog = vl_hog_new(VlHogVariantUoctti, 9, tr);
            const int sizes[][2] = {{64, 48}, {37, 29}, {64, 48}, {640, 480}};
            std::vector<Record> out;
            for (int i = 0; i < 4; ++i) out.push_back(put_image(hog, s + i, sizes[i][0], sizes[i][1], 1, 8, 9, 1, 0, tr));
            vl_hog_delete(hog);
            return out;
        });
    }
    // put_polar_field: W, H, cell size, K, variant, bilinear, transposed, directed
    const int polar[][8] = {
        {37, 29, 4, 9, 1, 0, 0, 1},  {37, 29, 4, 9, 1, 1, 1, 0},  {160, 120, 8, 16, 0, 1, 0, 0},
        {160, 120, 8, 4, 1, 0, 1, 1}, {55, 55, 11, 4, 0, 0, 1, 0}, {1920, 1080, 8, 9, 1, 1, 0, 1},
    };
    for (const auto& c : polar) {
        const int s = seed++;
        cases.push_back([=] { return std::vector<Record>{one_put_polar(s, c[0], c[1], c[2], c[3], c[4], c[5], c[6], c[7])}; });
    }
    // render: K {1, 4, 9, 16} x variant x transposed on random signed features, and the features of a put
    const int grids[][2] = {{1, 1}, {7, 5}, {13, 9}, {40, 30}};
    int gi = 0;
    for (int K : {1, 4, 9, 16})
        for (int variant = 0; variant < 2; ++variant)
            for (int tr = 0; tr < 2; ++tr) {
                const int s = seed++, w = grids[gi % 4][0], h = grids[gi % 4][1];
                ++gi;
                cases.push_back([=] { return std::vector<Record>{one_render(s, w, h, K, variant, tr, 0)}; });
            }
    for (int tr = 0; tr < 2; ++tr) {
        const int s = seed++;
        cases.push_back([=] { return std::vector<Record>{one_render(s, 20, 15, 9, 1, tr, 1)}; });
    }

    std::vector<std::vector<Record>> results(cases.size());
    if (argc > 2 && std::string(argv[2]) == "threads") {
        std::vector<std::thread> pool;
        for (int t = 0; t < 4; ++t)
            pool.emplace_back([&, t] {
                for (size_t i = t; i < cases.size(); i += 4) results[i] = cases[i]();
            });
        for (std::thread& th : pool) th.join();
    } else {
        for (size_t i = 0; i < cases.size(); ++i) results[i] = cases[i]();
    }
    FILE* f = std::fopen(argv[1], "wb");
    if (!f) return 1;
    size_t records = 0;
    for (const auto& rs : results)
        for (const Record& r : rs) {
            const int32_t n = (int32_t)r.ints.size();
            const int64_t m = (int64_t)r.data.size();
            std::fwrite(&n, sizeof(n), 1, f);
            std::fwrite(r.ints.data(), sizeof(int32_t), r.ints.size(), f);
            std::fwrite(&m, sizeof(m), 1, f);
            std::fwrite(r.data.data(), sizeof(float), r.data.size(), f);
            ++records;
        }
    std::fclose(f);
    std::printf("%zu records\n", records);
    return 0;
}
