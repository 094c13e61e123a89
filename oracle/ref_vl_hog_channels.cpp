// TEST INFRASTRUCTURE ONLY -- never linked into the product library.
//
// The reference's OWN hog.c (include/rcr/hog.h + hog.c of the reference tree, compiled where they lie by
// oracle/vl_hog_ref.py) with every input of vl_hog_put_image: a planar float image of num_channels channels (VLFeat's layout:
// channel k at image + k * width * height) and the bilinear orientation switch.  No reference source is copied into this
// repository.  Built to oracle/_ref/libref_vl_hog_channels.so (git-ignored).
extern "C" {
#include "hog.h"  // -I<reference>/include/rcr
}

extern "C" {

// vl_hog_new + vl_hog_set_use_bilinear_orientation_assignments + vl_hog_put_image + vl_hog_extract.  dims receives hogW,
// hogH, dd; out (dd * hogH * hogW floats, planar [dd][hogH][hogW]) may be NULL.  Returns 0 on success.
int ref_vl_hog_channels(int variant, int num_orientations, const float* image, int width, int height, int num_channels,
                        int cell_size, int bilinear, float* out, int* dims)
{
    VlHog* hog = vl_hog_new(variant == 0 ? VlHogVariantDalalTriggs : VlHogVariantUoctti, (vl_size)num_orientations, VL_FALSE);
    if (!hog) return 1;
    vl_hog_set_use_bilinear_orientation_assignments(hog, bilinear ? VL_TRUE : VL_FALSE);
    vl_hog_put_image(hog, image, (vl_size)width, (vl_size)height, (vl_size)num_channels, (vl_size)cell_size);
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
