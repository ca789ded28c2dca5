"""The CUDA raster kernel (every variant a step may launch: exact / fast fragment stage, with and without segmentation, any triangle-list
capacity and band count, any frame size) against the independent restatement of the rasterisation rules (raster_ref.py) on the
constructed scene families of raster_scenes.py.  Each scene first proves, from the restatement's record, that it reaches the branch it
was built for (test_raster_independent.py checks the same families against the oracle on the CPU).

  * unclipped scenes: coverage identical in every pixel, the winning instance identical (segmentation: instance i has tag i + 1), w to
    float32 rounding (relative 2e-5; at sizes other than 128 x 72 up to 8 pixels to 1e-4 and 8 pixels with another winner: long thin
    triangles at extreme aspect, near-equal depths of two instances);
  * clipped scenes: at most 8 pixels per 128 x 72 frame's worth differ (new clipper vertices in float32 and float64 can snap one
    sub-pixel apart; w near the far plane carries float32 rounding of 1 / w);
  * fast against exact: depth and segmentation byte-identical, colour within 1 LSB with more than 99.9 % of the bytes identical;
  * colour: the exact variant byte-identical to the oracle's rasteriser in colour and depth (every family, list capacity, band count
    and size); both variants against the float64 fragment stage (raster_ref.shade64) by raster_ref.colour_rule wherever the same
    instance won, with at least 99.9 % of the bytes equal to the float64 byte.

Variants run as a sparse matrix: every family at 128 x 72 in all four shading x segmentation variants; triangle-list capacity x band
count on a subset; other sizes up to the widest the API accepts (768) on a subset.  The off-screen envelope: triangles with a corner
2^18 .. 2^25 pixels beyond the frame just in front of the near plane must match wherever every snapped coordinate is below 2^30.5
sub-pixels and every difference of two corners below 2^31."""
import numpy as np
import pytest

import orc
import raster_ref as ref
import raster_scenes as scenes

pytestmark = pytest.mark.gpu


def _draw(view16, inst, W, H, fast=0, tri_cap=0, bands=0):
    from megaverse_b200 import capi

    rgba, depth, seg, stats = capi.render_instances(view16, inst, W, H, want_depth=True, fast=fast, segmentation=True, tri_cap=tri_cap, bands=bands, stats=True)
    return rgba, depth, seg, stats


def _check(family, R, out, W, H, fast, clipped=None):
    """out = (rgba, depth, seg, ...) of _draw for the scene R was drawn from"""
    rgba, depth, seg = out[:3]
    clipped = family in scenes.CLIPPED if clipped is None else clipped
    cov_dev, cov_ref = depth > 0, R.w > 0
    mism = int((cov_dev != cov_ref).sum())
    both = cov_dev & cov_ref
    rel = np.abs(depth[both].astype(np.float64) - R.w[both]) / R.w[both]
    assert np.array_equal(seg > 0, cov_dev), "segmentation 0 exactly where nothing was drawn"
    if not fast:  # the exact fragment stage reproduces the oracle's float32 arithmetic: colour and depth byte for byte
        o_rgba, o_depth = orc.render_instances(*R.scene, W, H, want_depth=True)
        assert np.array_equal(depth.view(np.uint32), o_depth.view(np.uint32)), "depth differs from the oracle's in %d pixels" % int((depth != o_depth).sum())
        assert np.array_equal(rgba, o_rgba), "colour differs from the oracle's in %d pixels" % int((rgba != o_rgba).any(-1).sum())
    # colour against the float64 fragment stage wherever the same instance won (raster_ref.colour_rule)
    same = both & (seg.astype(np.int32) == R.inst)
    broken, differ, worst, dmax = ref.colour_rule(R.frag, rgba, same, fast=bool(fast))
    print("%s %dx%d %s: %d colour bytes differ from the float64 ones (by up to %d), worst boundary margin among them %.4f LSB, %d break the "
          "rule" % (family, W, H, "fast" if fast else "exact", differ, dmax, worst, broken))
    if clipped:  # 8 pixels per 128 x 72 frame's worth of pixels
        allowed = max(8, 8 * W * H // (128 * 72))
        assert mism <= allowed, "coverage differs in %d pixels" % mism
        assert (rel > 1e-4).sum() <= allowed, "w differs in %d pixels" % int((rel > 1e-4).sum())
        assert broken <= 3 * allowed, "%d colour bytes break the rule (%d differ, by up to %d)" % (broken, differ, dmax)
        assert differ <= 0.001 * W * H * 3, "%d of the %d colour bytes differ from the float64 ones" % (differ, W * H * 3)
        return
    assert mism == 0, "coverage differs in %d pixels" % mism
    loose = 0 if (W, H) == (128, 72) else 8
    assert rel.max(initial=0) < 1e-4 and (rel > 2e-5).sum() <= loose, "depth differs by %.3g" % rel.max(initial=0)
    wrong = int((seg[cov_dev].astype(np.int32) != R.inst[cov_dev]).sum())  # (elsewhere near-equal depths of two instances may swap)
    assert wrong <= loose, "the winning instance differs in %d pixels" % wrong
    assert broken == 0, "%d colour bytes break the rule (%d differ, by up to %d; worst margin %.4f LSB)" % (broken, differ, dmax, worst)
    # of the frame's colour bytes (as fast against exact above), those where the same instance won equal the float64 byte
    assert differ <= 0.001 * W * H * 3, "%d of the %d colour bytes differ from the float64 ones" % (differ, W * H * 3)


@pytest.mark.parametrize("family", sorted(scenes.FAMILIES))
def test_every_family_every_variant_at_128x72(family):
    W, H = 128, 72
    view16, inst = scenes.build(family, W, H)
    R = ref.render(view16, inst, W, H)
    scenes.check_reach(family, R, W, H)
    from megaverse_b200 import capi

    exact, d_exact, s_exact, st = _draw(view16, inst, W, H, fast=0)
    fast, d_fast, s_fast, _ = _draw(view16, inst, W, H, fast=1)
    _check(family, R, (exact, d_exact, s_exact), W, H, fast=0)
    _check(family, R, (fast, d_fast, s_fast), W, H, fast=1)
    assert np.array_equal(d_exact.view(np.uint32), d_fast.view(np.uint32)) and np.array_equal(s_exact, s_fast), "fast and exact differ in depth or segmentation"
    diff = np.abs(exact.astype(np.int16) - fast.astype(np.int16))
    assert diff.max() <= 1 and (diff == 0).mean() > 0.999
    # segmentation off: the same colour and depth
    rgba_ns, d_ns = capi.render_instances(view16, inst, W, H, want_depth=True, fast=0)
    assert np.array_equal(rgba_ns, exact) and np.array_equal(d_ns.view(np.uint32), d_exact.view(np.uint32))
    if family in scenes.CLIPPED:
        assert st[4] > 0, "the kernel clipped items"


@pytest.mark.parametrize("tri_cap", [0, 96, 32])
@pytest.mark.parametrize("bands", [1, 2, 3])
@pytest.mark.parametrize("family", ["duplicates", "tiny_and_large", "edge_bounds", "borders", "highlights", "near_plane"])
def test_list_capacity_and_bands(family, tri_cap, bands):
    W, H = 128, 72
    kw = {"band_rows": [((H // 4 + bands - 1) // bands) * 4 * k for k in range(1, bands)]} if family == "borders" else {}
    view16, inst = scenes.build(family, W, H, **kw)
    R = ref.render(view16, inst, W, H)
    scenes.check_reach(family, R, W, H)
    out = _draw(view16, inst, W, H, tri_cap=tri_cap, bands=bands)
    _check(family, R, out, W, H, fast=0)
    st = out[3]
    if tri_cap == 32 and family in ("duplicates", "tiny_and_large", "highlights", "near_plane"):
        assert st[6] > bands, "views drawn in several list batches"


@pytest.mark.parametrize("gap", [130, 200])
def test_duplicates_across_instance_chunks_and_list_batches(gap):
    """copies of one box `gap` places apart, the first copy in the first 128-instance chunk and the second in a later one; with tri_cap 32
    and one band at least 32 drawn triangles lie between the two copies in draw order, so no list batch can hold both"""
    W, H = 128, 72
    view16, inst = scenes.build("duplicates", W, H, gap=gap)
    R = ref.render(view16, inst, W, H)
    n_boxes = int((inst[:, 0] == 0).sum())
    firsts = range(n_boxes - gap)   # copy j and j + gap
    seq = [p["inst"] for p in R.pieces]
    split = 0
    for j in firsts:
        won = int((R.inst == j + gap + 1).sum())
        if j >= 128 or j + gap < 128 or not won or j not in seq:
            continue
        between = sum(1 for i in seq if j < i < j + gap)
        split += between >= 32
        assert not (R.inst == j + 1).any() or won, "the later copy wins every tie"
    assert split >= 3, "pairs in different chunks, with at least 32 drawn triangles between the copies"
    for tri_cap, bands in ((0, 0), (32, 1)):
        out = _draw(view16, inst, W, H, tri_cap=tri_cap, bands=bands)
        _check("duplicates", R, out, W, H, fast=0)
        if tri_cap == 32:
            assert out[3][6] > 2


def test_far_clipping_matches_the_oracle_bit_for_bit():
    """the far-plane family once more, against the oracle's rasteriser, which clips in the same float32 arithmetic: colour and depth
    byte-identical.  The independent rules need a few pixels of slack where clipping creates vertices; this comparison needs none, so a
    far plane the clipper ignores (leaving the per-sample z <= 1 test to cut the triangle) shows even where it moves no whole pixel."""
    for W, H in ((128, 72), (160, 96)):
        for seed in range(3):
            view16, inst = scenes.build("far_plane", W, H, seed=seed)
            rgba, depth, _, st = _draw(view16, inst, W, H, fast=0)
            o_rgba, o_depth = orc.render_instances(view16, inst, W, H, want_depth=True)
            assert st[4] > 0
            assert np.array_equal(depth.view(np.uint32), o_depth.view(np.uint32)), "depth differs in %d pixels" % int((depth != o_depth).sum())
            assert np.array_equal(rgba, o_rgba), "colour differs in %d pixels" % int((rgba != o_rgba).any(-1).sum())


SIZES = [(64, 64), (160, 96), (32, 512), (512, 32), (768, 432), (768, 32)]


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("family", ["ties", "borders", "tiny_and_large", "far_plane", "mirrored", "grazing", "edge_bounds", "slivers", "highlights",
                                    "scaled_normals", "near_plane", "palette"])
def test_other_sizes(family, size):
    W, H = size
    view16, inst = scenes.build(family, W, H)
    R = ref.render(view16, inst, W, H)
    scenes.check_reach(family, R, W, H)
    for fast in (1, 0):
        _check(family, R, _draw(view16, inst, W, H, fast=fast), W, H, fast=fast)


@pytest.mark.parametrize("W,H", [(128, 72), (768, 32)])
@pytest.mark.parametrize("opposite", [False, True])
def test_offscreen_vertex_envelope(W, H, opposite):
    """a corner 2^k pixels beyond the frame (k = 18 .. 25 in quarter steps), just in front of the near plane: the kernel must match the
    guard-band answer whenever every snapped coordinate is below 2^30.5 sub-pixels and every difference of two corners below 2^31 (then
    positions and coefficients fit int32, edge constants and bounds int64).  Beyond, the mismatches are reported (int32 saturation of the
    snap, wrap of the edge coefficients); the scenes must reach within a quarter octave of both limits."""
    found = []
    for k in np.arange(18.0, 25.01, 0.25):
        view16, inst = scenes.offscreen_vertex(W, H, k, opposite)
        R = ref.render(view16, inst, W, H)
        top, delta = max(t["max_coord"] for t in R.tris), max(t["max_delta"] for t in R.tris)
        _, depth, seg, _ = _draw(view16, inst, W, H)
        mism = int(((depth > 0) != (R.w > 0)).sum())
        inside = top < 2.0 ** 30.5 and delta < 2.0 ** 31
        found.append((k, top, delta, mism, inside))
        if inside:
            assert mism == 0, "2^%.2f px off-screen (|s| = 2^%.2f, |ds| = 2^%.2f): coverage differs in %d pixels" % (k, np.log2(top), np.log2(delta), mism)
    print("\n%dx%d %s: " % (W, H, "opposite sides" if opposite else "one side") +
          ", ".join("2^%.2f px |s| 2^%.2f |ds| 2^%.2f: %d px differ" % (k, np.log2(t), np.log2(d), m) for k, t, d, m, _ in found))
    largest = max((t, d) for _, t, d, _, ok in found if ok)
    assert largest[0] > 2.0 ** 30.25 or largest[1] > 2.0 ** 30.75, "the scenes come close to the envelope's edge"


def test_frames_wider_than_the_envelope_are_refused():
    from megaverse_b200 import capi

    view16, inst = scenes.build("ties", 800, 32)
    with pytest.raises(capi.MegaverseError):
        capi.render_instances(view16, inst, 800, 32, fast=1)
    with pytest.raises(capi.MegaverseError):
        capi.Engine("Collect", 1, 1, 800, 4)
