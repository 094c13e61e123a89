// TEST INFRASTRUCTURE ONLY -- never linked into the product library.
//
// The reference's OWN hog.c (include/rcr/hog.h + hog.c of the reference tree, compiled where they lie by
// oracle/vl_hog_polar_ref.py) through vl_hog_put_polar_field: a caller's gradient field, modulus and angle per pixel, with the
// directed and bilinear orientation switches.  No reference source is copied into this repository.  Built to
// oracle/_ref/libref_vl_hog_polar.so (git-ignored).
extern "C" {
#include "hog.h"  // -I<reference>/include/rcr
}

extern "C" {

// vl_hog_new + vl_hog_set_use_bilinear_orientation_assignments + vl_hog_put_polar_field + vl_hog_extract of one field (modulus
// and angle, width x height floats each, row-major).  dims receives hogW, hogH, dd; out (dd * hogH * hogW floats, planar
// [dd][hogH][hogW]) may be NULL.  Returns 0 on success.
int ref_vl_hog_polar(int variant, int num_orientations, const float* modulus, const float* angle, int width, int height,
                     int directed, int cell_size, int bilinear, float* out, int* dims)
{
    VlHog* hog = vl_hog_new(variant == 0 ? VlHogVariantDalalTriggs : VlHogVariantUoctti, (vl_size)num_orientations, VL_FALSE);
    if (!hog) return 1;
    vl_hog_set_use_bilinear_orientation_assignments(hog, bilinear ? VL_TRUE : VL_FALSE);
    vl_hog_put_polar_field(hog, modulus, angle, directed ? VL_TRUE : VL_FALSE, (vl_size)width, (vl_size)height, (vl_size)cell_size);
    if (dims) {
        dims[0] = (int)vl_hog_get_width(hog);
        dims[1] = (int)vl_hog_get_height(hog);
        dims[2] = (int)vl_hog_get_dimension(hog);
    }
    if (out) vl_hog_extract(hog, out);
    vl_hog_delete(hog);
    return 0;
}

}  // extern "C"
