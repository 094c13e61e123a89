"""The hog.h drop-in (superviseddescent_b200/include/rcr/hog.h) and its host tables, without a GPU.

  - sd_hog_permutation and sd_hog_glyphs (through vl_hog_permutation / vl_hog_glyphs) equal the permutation and glyphs of the
    reference's own vl_hog_new, element for element, for K = 1..16, both variants, transposed and not;
  - the shell compiles with -std=c++14 -Wall on its own, and with rcr/adaptive_vlhog.hpp in one translation unit
    (tests/cpp/test_hog_h.cpp), and refuses what hog.c asserts and what this project does not support with std::runtime_error;
  - the driver program oracle/vl_hog_driver.cpp compiles against the reference's hog.h and against the shell."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = ["-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "superviseddescent_b200", "include")]


@pytest.fixture(scope="module")
def lib_dir():
    from superviseddescent_b200 import build
    return os.path.dirname(build.build())


@pytest.fixture(scope="module")
def ref(oracle):
    from oracle import vl_hog_api_ref
    vl_hog_api_ref.build()
    if not vl_hog_api_ref.available():
        pytest.skip("oracle/_ref (the reference's hog.c) is not built")
    return vl_hog_api_ref


def _compile(args, lib_dir, out):
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type"] + INC + args + ["-L", lib_dir, "-lsd_b200",
                                                                                     f"-Wl,-rpath,{lib_dir}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    assert "warning" not in r.stderr, r.stderr[-4000:]


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("transposed", [False, True])
def test_host_tables_are_hog_c(ref, variant, transposed, lib_dir):
    from superviseddescent_b200 import api
    for K in range(1, 17):
        hog = ref.Hog(variant, K, transposed)
        assert np.array_equal(api.vl_hog_permutation(variant, K), hog.permutation()), K
        glyphs = api.vl_hog_glyphs(K, transposed)
        assert glyphs.shape == (K, 21, 21)
        assert np.array_equal(glyphs.view(np.uint32), hog.glyphs().view(np.uint32)), K


def test_host_tables_refuse_out_of_range(lib_dir):
    from superviseddescent_b200 import api
    for K in (0, 17):
        with pytest.raises(ValueError):
            api.vl_hog_permutation(1, K)
        with pytest.raises(ValueError):
            api.vl_hog_glyphs(K)


def test_shell_compiles_alone(lib_dir, tmp_path):
    src = tmp_path / "alone.cpp"
    src.write_text('#include "rcr/hog.h"\nint main() { VlHog* h = vl_hog_new(VlHogVariantUoctti, 9, VL_FALSE); '
                   'int d = (int)vl_hog_get_dimension(h); vl_hog_delete(h); return d == 31 ? 0 : 1; }\n')
    _compile([str(src)], lib_dir, str(tmp_path / "alone"))


def test_shell_with_adaptive_vlhog_refuses_with_runtime_error(lib_dir, tmp_path):
    out = str(tmp_path / "test_hog_h")
    _compile([os.path.join(ROOT, "tests", "cpp", "test_hog_h.cpp")], lib_dir, out)
    r = subprocess.run([out], capture_output=True, text=True, timeout=120)
    print(r.stdout)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


def test_driver_compiles_against_both(ref, lib_dir, tmp_path):
    assert os.path.exists(ref.DRIVER)
    _compile([os.path.join(ROOT, "oracle", "vl_hog_driver.cpp")], lib_dir, str(tmp_path / "driver_shell"))
