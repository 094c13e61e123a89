// TEST INFRASTRUCTURE ONLY -- never linked into the product library.
//
// The reference's OWN hog.c (include/rcr/hog.h + hog.c of the reference tree, compiled where they lie by
// oracle/vl_hog_api_ref.py) through its VlHog object: vl_hog_new with the transposed switch, put_image and put_polar_field,
// render of caller-given features into a caller-given image, and the object's permutation and glyphs.  No reference source is
// copied into this repository.  Built to oracle/_ref/libref_vl_hog_api.so (git-ignored).
extern "C" {
#include "hog.h"  // -I<reference>/include/rcr
}

#include <cstring>

extern "C" {

void* ref_hog_new(int variant, int num_orientations, int transposed, int bilinear)
{
    VlHog* h = vl_hog_new(variant == 0 ? VlHogVariantDalalTriggs : VlHogVariantUoctti, (vl_size)num_orientations,
                          transposed ? VL_TRUE : VL_FALSE);
    vl_hog_set_use_bilinear_orientation_assignments(h, bilinear ? VL_TRUE : VL_FALSE);
    return h;
}

void ref_hog_delete(void* h) { vl_hog_delete((VlHog*)h); }

void ref_hog_put_image(void* h, const float* image, int width, int height, int channels, int cell_size)
{
    vl_hog_put_image((VlHog*)h, image, (vl_size)width, (vl_size)height, (vl_size)channels, (vl_size)cell_size);
}

void ref_hog_put_polar(void* h, const float* modulus, const float* angle, int directed, int width, int height, int cell_size)
{
    vl_hog_put_polar_field((VlHog*)h, modulus, angle, directed ? VL_TRUE : VL_FALSE, (vl_size)width, (vl_size)height, (vl_size)cell_size);
}

// dims: hogW, hogH, dd (of the last put), glyph size
void ref_hog_dims(void* h, int* dims)
{
    dims[0] = (int)vl_hog_get_width((VlHog*)h);
    dims[1] = (int)vl_hog_get_height((VlHog*)h);
    dims[2] = (int)vl_hog_get_dimension((VlHog*)h);
    dims[3] = (int)vl_hog_get_glyph_size((VlHog*)h);
}

void ref_hog_extract(void* h, float* out) { vl_hog_extract((VlHog*)h, out); }

// vl_hog_render of features [dd][height][width] into image (height * glyph rows of width * glyph floats), read-modify-write
void ref_hog_render(void* h, float* image, const float* features, int width, int height)
{
    vl_hog_render((VlHog*)h, image, features, (vl_size)width, (vl_size)height);
}

void ref_hog_permutation(void* h, long long* out)
{
    const VlHog* hog = (const VlHog*)h;
    std::memcpy(out, vl_hog_get_permutation(hog), sizeof(long long) * vl_hog_get_dimension(hog));
}

void ref_hog_glyphs(void* h, float* out)
{
    const VlHog* hog = (const VlHog*)h;
    std::memcpy(out, hog->glyphs, sizeof(float) * hog->glyphSize * hog->glyphSize * hog->numOrientations);
}

}  // extern "C"
