// The hog.h drop-in next to the adaptive_vlhog.hpp shell in one translation unit (the reference includes hog.h from
// adaptive_vlhog.hpp inside extern "C" { }), and the calls it refuses.  Every refusal below happens before any device work, so
// this program runs with or without a GPU: it prints one line per refused call and "ALL OK" when each one threw
// std::runtime_error.
#include "rcr/adaptive_vlhog.hpp"
extern "C" {
#include "rcr/hog.h"
}

#include <cstdio>
#include <functional>
#include <stdexcept>
#include <string>
#include <vector>

static int failures = 0;

static void expect_throw(const char* what, const std::function<void()>& f)
{
    try {
        f();
        std::printf("FAIL %s: no exception\n", what);
        ++failures;
    } catch (const std::runtime_error& e) {
        std::printf("ok   %s: %s\n", what, e.what());
    }
}

int main()
{
    const rcr::HoGParam param{VlHogVariantUoctti, 5, 8, 9, 0.1f};   // the shell's HoGParam sees hog.h's VlHogVariant
    (void)param;
    std::vector<float> img(64 * 64 * 17, 1.f), feat(40 * 4 * 4, 0.f), out(21 * 21 * 16, 0.f);
    expect_throw("numOrientations 0", [] { vl_hog_new(VlHogVariantUoctti, 0, VL_FALSE); });
    expect_throw("numOrientations 17", [] { vl_hog_new(VlHogVariantDalalTriggs, 17, VL_FALSE); });
    VlHog* hog = vl_hog_new(VlHogVariantUoctti, 9, VL_FALSE);
    if (vl_hog_get_dimension(hog) != 31 || vl_hog_get_glyph_size(hog) != 21 || vl_hog_get_width(hog) != 0 || vl_hog_get_height(hog) != 0) {
        std::printf("FAIL dimension / glyph size / empty grid\n");
        ++failures;
    }
    expect_throw("extract before put", [&] { vl_hog_extract(hog, out.data()); });
    expect_throw("cell size 33", [&] { vl_hog_put_image(hog, img.data(), 64, 64, 1, 33); });
    expect_throw("cell size 0", [&] { vl_hog_put_image(hog, img.data(), 64, 64, 1, 0); });
    expect_throw("width 3", [&] { vl_hog_put_image(hog, img.data(), 3, 64, 1, 4); });
    expect_throw("less than half a cell", [&] { vl_hog_put_image(hog, img.data(), 6, 64, 1, 16); });
    expect_throw("17 channels", [&] { vl_hog_put_image(hog, img.data(), 64, 64, 17, 8); });
    expect_throw("0 channels", [&] { vl_hog_put_image(hog, img.data(), 64, 64, 0, 8); });
    expect_throw("null image", [&] { vl_hog_put_image(hog, nullptr, 64, 64, 1, 8); });
    expect_throw("polar cell size 33", [&] { vl_hog_put_polar_field(hog, img.data(), img.data(), VL_TRUE, 64, 64, 33); });
    expect_throw("polar null angle", [&] { vl_hog_put_polar_field(hog, img.data(), nullptr, VL_TRUE, 64, 64, 8); });
    expect_throw("render width 0", [&] { vl_hog_render(hog, out.data(), feat.data(), 0, 1); });
    expect_throw("render null image", [&] { vl_hog_render(hog, nullptr, feat.data(), 1, 1); });
    vl_hog_set_use_bilinear_orientation_assignments(hog, VL_TRUE);
    if (!vl_hog_get_use_bilinear_orientation_assignments(hog)) {
        std::printf("FAIL bilinear switch\n");
        ++failures;
    }
    vl_hog_delete(hog);
    if (failures) return 1;
    std::printf("ALL OK\n");
    return 0;
}
