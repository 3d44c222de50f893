"""CPU checks of the polygon edge inputs (tests/polygon_edge_inputs.py) and of the oracle
test_gpu_polygon_edges.py holds mrx_poly_decode to: each builder really holds the edge it is
named for (counted), each oracle variant -- a model of one mutant of tools/mutate_polygons.py --
changes the expected masks on the GPU test's own inputs, the windowed walk equals the dense one,
the host's toggle bucket bound covers every part, and no toggle inside the image comes from the
pair where two edges meet."""
import numpy as np
import pytest

import polygon_edge_inputs as pe
import polygon_oracle as po
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import pack_polygons


def _geom(H, W):
    return [H, W, H, W, 0, 0, H, W]


@pytest.fixture(scope="module")
def built():
    return {b.__name__: b() for b in pe.BUILDERS}


@pytest.fixture(scope="module")
def counts(built):
    return {name: pe.census(d["images"]) for name, d in built.items()}


@pytest.mark.parametrize("name", [b.__name__ for b in pe.BUILDERS])
def test_builder_holds_its_edge(built, counts, name):
    short = {k: (counts[name][k], want) for k, want in built[name]["expect"].items()
             if counts[name][k] < want}
    assert not short, short


def test_search_covers_every_branch():
    """x-major and y-major walks, forwards and backwards, a >= 0 and a < 0: three parts each."""
    for variant in ("fused", "recip"):
        found = pe.search_minor(variant)
        assert len(found) == 8 and all(len(v) == 3 for v in found.values()), variant


def test_fused_minor_is_a_live_trap():
    """The issue's smallest case: a = 3, s = -5/6, t = 3 gives 1 with one rounding per operation
    and 0 as an FMA, since -5/6 * 3 rounds to -2.5 exactly."""
    assert po._minor(3, -5 / 6, 3, False) == 1 and po._minor(3, -5 / 6, 3, True) == 0


@pytest.mark.parametrize("variant", sorted(pe.VARIANTS))
def test_variant_changes_expected_masks(counts, variant):
    assert sum(c[variant + "_instances"] for c in counts.values()) > 0


def test_variants_default_off():
    """With no keyword the oracle is pycocotools' (tests/test_polygon_oracle.py); every variant
    switched off explicitly gives the same runs."""
    rng = np.random.default_rng(4)
    for _ in range(30):
        xy = [float(v) for v in np.round(rng.uniform(-3, 25, 10) * 5) / 5]
        want = po.fr_poly(xy, 17, 23)
        assert po.fr_poly(xy, 17, 23, fused=False, recip=False, floor=False, row_up=False,
                          clamp_h1=False, xmaj_first=False, row_late=False) == want


def _sweep(seed, n):
    """Seeded parts of every grid (real, 0.2, 1, 0.5) around small images."""
    rng = np.random.default_rng(seed)
    out = []
    for it in range(n):
        H, W = int(rng.integers(1, 40)), int(rng.integers(1, 40))
        step = [0, 0.2, 1, 0.5][it % 4]
        xy = rng.uniform(-5, max(H, W) + 5, 2 * int(rng.integers(3, 8)))
        if step:
            xy = np.round(xy / step) * step
        out.append(((H, W), [float(v) for v in xy]))
    return out


def _small_parts(built):
    for name, d in built.items():
        if name == "int_range":
            continue
        for (H, W), segms in d["images"]:
            for segm in segms:
                if not pe.is_boxes(segm):
                    for xy in segm:
                        yield (H, W), xy
    yield from _sweep(5, 1500)


def test_windowed_walk_equals_dense(built):
    for (H, W), xy in _small_parts(built):
        x, y = po.scaled_vertices(xy)
        dense = po.toggles(*po.walk(x, y), H, W)
        win = po.toggles(*po.walk(x, y, window=(-3, 5 * W + 3)), H, W)
        assert [t[:2] + t[3:] for t in win] == [t[:2] + t[3:] for t in dense], (H, W, xy)


def test_toggle_bound_covers_every_part(built):
    """pack_polygons' part_tog span, min(W, (|dx| + 2) // 5 + 1) + 1 per edge, is at least the
    oracle's in-image toggle count of every part; the tighter min(W, (|dx| + 4) // 5) per edge
    also holds (census asserts it per edge) and the dense inputs reach it."""
    slack = []
    cases = [(hw, [[xy]]) for hw, xy in _sweep(6, 600)]
    for d in built.values():
        cases += d["images"]
    for (H, W), segms in cases:
        pk = pack_polygons([_geom(H, W)], [np.ones(len(segms), np.int32)], [segms])
        span = np.diff(pk["part_tog"])
        p = 0
        for segm in segms:
            parts = segm if not pe.is_boxes(segm) else [
                [x, y, x, y + h, x + w, y + h, x + w, y] for x, y, w, h in segm]
            for xy in parts:
                got = len(po.part_toggles(xy, H, W, window=True))
                assert got <= span[p], (H, W, xy, got, span[p])
                slack.append(int(span[p]) - got)
                p += 1
    print(f"toggle bucket slack: smallest {min(slack)} over {len(slack)} parts")
    assert min(slack) >= 1      # the junction's + 1 per edge is never used
    dense = pe.census(pe.dense_toggles()["images"], variants=False)
    assert dense["tight_edges"] >= 60 and dense["wide_edges"] >= 6


def test_no_junction_toggle_and_no_odd_column(counts):
    """Where edge j - 1 ends and edge j begins, both emit u = x exactly at a vertex with x >= 0:
    an x-major edge's u is xs + t, and a y-major edge's end is (int)(x + .5 + e) with |e| far
    below .5.  At a vertex with x < 0 both u are x or x + 1, at most 0, so xd < 2 = 5*0 + 2.
    Either way the junction pair never toggles a column inside the image: the kernel's junction
    branch emits nothing there, and the + 1 per edge of the host bound is slack.  And every
    column holds an even number of toggles (the closed walk crosses u = c + 1/2 an even number
    of times, each crossing a pair with |du| = 1), so a part's carry into the next pass of the
    column scan is 0."""
    for name, c in counts.items():
        assert c["junction"] == 0 and c["odd_columns"] == 0, name
    n = pe.census([(hw, [[xy]]) for hw, xy in _sweep(7, 3000)], variants=False)
    assert n["junction"] == 0 and n["odd_columns"] == 0
    assert n["row_0"] + n["row_H"] > 1000


def test_int_range_ends_accepted_one_past_refused():
    ((H, W), segms), = pe.int_range()["images"]
    pk = pack_polygons([_geom(H, W)], [np.ones(len(segms), np.int32)], [segms])
    v = pk["vert"].astype(np.int64)
    assert v.max() == pe.INT_MAX and v.min() == pe.INT_MIN
    for bad, match in zip(pe.int_range_refused(), ["does not fit", "does not fit",
                                                    "differ by more", "differ by more"]):
        with pytest.raises(ValueError, match=match):
            pack_polygons([_geom(H, W)], [np.ones(1, np.int32)], [[bad]])


def test_big_image_positions_pass_2_31():
    ((H, W), segms), = pe.big_image()["images"]
    assert H * W >= 1 << 31
    runs = po.ann_to_rle(segms[0], H, W, window=True)
    assert sum(runs) == H * W and sum(runs[:-1]) > 1 << 31
