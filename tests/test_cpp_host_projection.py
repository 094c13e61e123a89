"""The C++14 shells' host batch projections (tests/cpp/test_host_projection.cpp), and the host callback type from plain C.

CPU: the translation units compile (the shell test as C++14; a C99 and a C++14 file that define an sd_host_project_fn, fill an
sd_level_host_projection and link against the library).  GPU: the pose example through rowwise(...) matches the plain-functor
route within the pose suite's bars, a class with project_host trains in chunks and tests, and exceptions come out of train() /
test()."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CALLBACK_SRC = r"""
#include "sd_b200.h"

/* columns [0, D) of each staged row, D from the user pointer */
static int ones(void* user, int level, const float* h_x, int64_t ldx, int64_t first_row, int rows, float* h_out, int64_t ld_out)
{
    const int D = *(const int*)user;
    int r, c;
    (void)level; (void)h_x; (void)ldx; (void)first_row;
    for (r = 0; r < rows; ++r)
        for (c = 0; c < D; ++c) h_out[(int64_t)r * ld_out + c] = 1.0f;
    return 0;
}

int train_with_ones(sd_ctx* ctx, const float* d_x, const float* d_gt, int n, int P, const sd_regulariser* reg, float* d_chunk,
                    int64_t ld, float* d_X, float* d_next)
{
    int D = 8;
    sd_level_host_projection proj;
    proj.fn = ones;
    proj.user = &D;
    proj.level = 0;
    proj.feature_length = D;
    proj.stage_half_bytes = 0;
    if (sd_train_level_host_projected(ctx, 0, &proj, d_x, d_gt, n, P, n, 0, 0, 0, reg, 0, d_chunk, ld, n, d_X, d_next, 0)) return 1;
    return sd_apply_level_host_projected(ctx, &proj, d_x, n, P, 0, 0, 0, d_X, d_chunk, ld, n, d_next);
}

int main(void) { return 0; }
"""


def _compile(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]


@pytest.fixture(scope="module")
def lib_dir():
    from superviseddescent_b200 import build
    return os.path.dirname(build.build())


@pytest.fixture(scope="module")
def host_projection_binary(tmp_path_factory, lib_dir):
    out = str(tmp_path_factory.mktemp("cpp") / "test_host_projection")
    _compile(["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
              "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_host_projection.cpp"),
              "-L", lib_dir, "-lsd_b200", f"-Wl,-rpath,{lib_dir}", "-lpthread", "-o", out])
    return out


def test_host_projection_compiles_as_cxx14(host_projection_binary):
    assert os.path.exists(host_projection_binary)


@pytest.mark.parametrize("compiler,std,ext", [("gcc", "-std=c99", "c"), ("g++", "-std=c++14", "cpp")])
def test_host_callback_type_is_usable_from_c_and_cxx14(tmp_path, lib_dir, compiler, std, ext):
    src = tmp_path / f"host_callback.{ext}"
    src.write_text(CALLBACK_SRC)
    out = str(tmp_path / f"host_callback_{ext}")
    _compile([compiler, std, "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-L", lib_dir,
              "-lsd_b200", f"-Wl,-rpath,{lib_dir}", "-o", out])
    assert os.path.exists(out)


@pytest.mark.gpu
def test_shell_host_projection_trains_and_tests(host_projection_binary):
    r = subprocess.run([host_projection_binary], capture_output=True, text=True, timeout=900)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    assert "POSE" in r.stdout and "CHUNKS" in r.stdout
    assert "RETHROWN project_host" in r.stdout and "RETHROWN rowwise" in r.stdout
