"""The C++14 shells' device batch projections (tests/cpp/test_projection.cpp), and the callback type from plain C.

CPU: the translation units compile (the shell test as C++14; a C99 and a C++14 file that define an sd_project_fn, fill an
sd_level_projection and link against the library).  GPU: a projection that writes HOG rows through the callback trains and tests
bit for bit as the HogTransform cascade, in one chunk and in chunks, and its exception comes out of train()."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CALLBACK_SRC = r"""
#include "sd_b200.h"

/* columns [0, D) of each row, D from the user pointer: the level's targets sit in the columns after them */
static int zeros(void* user, sd_ctx* ctx, int level, const float* d_x, int64_t ldx, int64_t first_row, int rows, float* d_out,
                 int64_t ld)
{
    const int D = *(const int*)user;
    int r, rc = 0;
    (void)level; (void)d_x; (void)ldx; (void)first_row;
    for (r = 0; r < rows && !rc; ++r) rc = sd_memset(ctx, d_out + (int64_t)r * ld, 0, (size_t)D * sizeof(float));
    return rc;
}

int train_with_zeros(sd_ctx* ctx, const float* d_x, const float* d_gt, int n, int P, const sd_regulariser* reg, float* d_chunk,
                     int64_t ld, float* d_X, float* d_next)
{
    int D = 8;
    sd_level_projection proj;
    proj.fn = zeros;
    proj.user = &D;
    proj.level = 0;
    proj.feature_length = D;
    if (sd_train_level_projected(ctx, 0, &proj, d_x, d_gt, n, P, n, 0, 0, 0, reg, 0, d_chunk, ld, n, d_X, d_next, 0)) return 1;
    return sd_apply_level_projected(ctx, &proj, d_x, n, P, 0, 0, 0, d_X, d_chunk, ld, n, d_next);
}

void* stream_of(const sd_ctx* ctx) { return sd_ctx_stream(ctx); }

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
def projection_binary(tmp_path_factory, lib_dir):
    out = str(tmp_path_factory.mktemp("cpp") / "test_projection")
    _compile(["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
              "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_projection.cpp"),
              "-L", lib_dir, "-lsd_b200", f"-Wl,-rpath,{lib_dir}", "-lpthread", "-o", out])
    return out


def test_projection_compiles_as_cxx14(projection_binary):
    assert os.path.exists(projection_binary)


@pytest.mark.parametrize("compiler,std,ext", [("gcc", "-std=c99", "c"), ("g++", "-std=c++14", "cpp")])
def test_callback_type_is_usable_from_c_and_cxx14(tmp_path, lib_dir, compiler, std, ext):
    src = tmp_path / f"callback.{ext}"
    src.write_text(CALLBACK_SRC)
    out = str(tmp_path / f"callback_{ext}")
    _compile([compiler, std, "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-L", lib_dir,
              "-lsd_b200", f"-Wl,-rpath,{lib_dir}", "-o", out])
    assert os.path.exists(out)


@pytest.mark.gpu
def test_shell_batch_projection_is_the_hog_level(projection_binary, golden):
    r = subprocess.run([projection_binary, golden.model_path], capture_output=True, text=True, timeout=600)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    assert r.stdout.count("IDENTICAL chunk") == 2 and "RETHROWN" in r.stdout
