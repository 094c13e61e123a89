"""The angle-to-bin rule of vl_hog_put_polar_field, restated without hog.c's loop (tests/polar_fields.py, the rule the device
applies), against the reference's own hog.c (oracle.vl_hog_polar_ref.vl_hog_polar).

hog.c brings floor(ho) into range with `while (bino < 0) bino += 2K` and then takes it modulo K or 2K; the device takes the
Euclidean residue with floorf and fmodf.  Fields with a single voting pixel run through hog.c at every angle of the sweep
(exact half steps, exact multiples, magnitudes up to 1e7, negative angles), for K = 1..16, directed and undirected:
  - nearest bin: the features equal, bit for bit, those of the same pixel at an angle inside the restated bin, away from its
    edges, which pins the residue and the tie rule (a tie goes to bino + 1);
  - bilinear: the directed dimensions that hog.c fills are exactly the restated pair."""
import numpy as np
import pytest

from polar_fields import angle_sweep, half_steps, polar_bins, polar_ho

CS, SIZE, PIXEL = 4, 12, (5, 6)          # a 3 x 3 cell grid, one voting pixel inside the centre cell


@pytest.fixture(scope="module")
def ref(oracle):
    from oracle import vl_hog_polar_ref
    vl_hog_polar_ref.build()
    if not vl_hog_polar_ref.available():
        pytest.skip("oracle/_ref (the reference's hog.c) is not built")
    return vl_hog_polar_ref


def _one_pixel(ref, angle, K, directed, bilinear):
    m = np.zeros((SIZE, SIZE), np.float32)
    a = np.zeros((SIZE, SIZE), np.float32)
    m[PIXEL] = 1.5
    a[PIXEL] = angle
    return ref.vl_hog_polar(m, a, CS, K, 1, directed, bilinear)


def test_half_steps_land_on_ties():
    """Most half steps (b + 0.5) pi / K have a float32 angle whose ho is exactly b + 0.5, so the sweep holds real ties."""
    for K in range(1, 17):
        halves, tried = half_steps(K)
        assert len(halves) >= tried // 2, (K, len(halves), tried)
        ho = polar_ho(halves, K)
        assert np.all(ho - np.floor(ho) == np.float32(0.5))


@pytest.mark.parametrize("K", range(1, 17))
@pytest.mark.parametrize("directed", [False, True])
def test_restated_bin_rule_is_hog_c(ref, K, directed):
    angles = angle_sweep(K)
    near, b0, b1, wo2 = polar_bins(angles, K, directed)
    period = 2 * K if directed else K
    assert np.all((near >= 0) & (near < period)) and np.all((b0 >= 0) & (b0 < period)) and np.all((b1 >= 0) & (b1 < period))
    centre = np.array([(c + 0.25) * np.pi / K for c in range(period)], dtype=np.float32)
    assert np.array_equal(polar_bins(centre, K, directed)[0], np.arange(period))
    canonical = {c: _one_pixel(ref, centre[c], K, directed, False) for c in range(period)}
    ties = 0
    for i, t in enumerate(angles):
        got = _one_pixel(ref, t, K, directed, False)
        assert np.array_equal(got, canonical[int(near[i])]), (K, directed, float(t), int(near[i]))
        ho = polar_ho(t, K)
        ties += bool(ho - np.floor(ho) == np.float32(0.5))
        # bilinear: the directed dimensions (UoCTTI: the first 2K) that hold a vote are the restated pair
        feats = _one_pixel(ref, t, K, directed, True)
        filled = {d for d in range(2 * K) if np.any(feats[d] > 0)}
        want = {int(b0[i])} | ({int(b1[i])} if wo2[i] > 0 else set())
        assert filled == want, (K, directed, float(t), filled, want)
    assert ties >= K
