"""The JPEG oracle and the files of tests/jpeg_edge_inputs.py: each builder's stated edge counts
recomputed from its files, the oracle held to the committed golden decodes (cv2.imdecode, recorded
with the versions and the CPU in tests/golden/jpeg_edges.npz) and to live cv2.imdecode where the
host runs libjpeg-turbo's x86-64 AVX2 code, every one-mistake variant of the IDCT shown to change
the expected pixels, and refusal parity."""
import functools
import hashlib
import os
import platform

import numpy as np
import pytest

import jpeg_edge_inputs as E
import jpeg_inputs as JI
import jpeg_oracle as O
import jpeg_progressive_oracle as PO
from matterport_maskrcnn_with_tensorflow_serving_b200 import jpeg as J

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_edges.npz")


@functools.lru_cache(maxsize=None)
def cases():
    base = E.all_cases()
    return base + E.progressive(base)


@functools.lru_cache(maxsize=None)
def golden():
    g = np.load(GOLDEN)
    return {k: g[k] for k in g.files}


def _is_avx2_x86():
    if platform.machine() not in ("x86_64", "AMD64"):
        return False
    try:
        with open("/proc/cpuinfo") as f:
            return " avx2" in f.read()
    except OSError:
        return False


def _oracle(blob):
    return (PO if J._frame_marker(blob) == 0xC2 else O).decode(blob)


@functools.lru_cache(maxsize=None)
def _oracle_of(name):
    c = {c.name: c for c in cases()}[name]
    try:
        return _oracle(c.blob)
    except J.JpegError as e:
        return e


def _scan(blob):
    hd = J.parse(blob)
    end = len(blob) - 2
    return blob[hd.scan_off:end]


def census(case):
    """The edge counts of a baseline file, recomputed from its bytes through the oracle's
    coefficient walk (keys as the builders state them)."""
    blob = case.blob
    out = {}
    try:
        hd = J.parse(blob)
    except J.JpegError as e:
        if "DC symbol above 15" in str(e):
            out["dc_symbol_16"] = 1
        return out
    trace = {}
    try:
        coef, hd = O.coefficients(blob, trace)
    except J.JpegError as e:
        if "overflows int32" in str(e):
            out["dc_int32_refused"] = 1
        return out
    comp_of = [0] if hd.ncomp == 1 else [ci for ci, (h, v) in enumerate(hd.samp)
                                         for _ in range(h * v)]
    comps = np.asarray(comp_of * (coef.shape[0] // hd.bpm))
    c = coef.astype(np.int64).reshape(-1, 8, 8)
    q = np.stack([hd.tables[ci][2] for ci in comps]).astype(np.int64).reshape(-1, 8, 8)
    x = O._w16(c * q)
    raw_ac = c[:, 1:, :].any(axis=(1, 2))
    dc_only = ~raw_ac & ~c[:, 0, 1:].any(axis=1)
    for v in (8191, 8192, 8193, -8191, -8192, -8193):
        out[f"dc_dq_{v}"] = int((dc_only & (c[:, 0, 0] * q[:, 0, 0] == v)).sum())
    full = raw_ac
    sums = [x[full, 0] + x[full, 4], x[full, 0] - x[full, 4], x[full, 7] + x[full, 3],
            x[full, 5] + x[full, 1]]
    out["sum_inside"] = sum(int(np.isin(s, (32767, -32768)).sum()) for s in sums)
    out["sum_wraps"] = sum(int(np.isin(s, (32768, -32769)).sum()) for s in sums)
    cols = O._one_d_simd(*[x[full, k, :] for k in range(8)], sum16=O._w16)
    p1 = np.stack([O._w32(v + 1024) >> 11 for v in cols])
    out["p1_over"] = int(((p1 > 32767) | (p1 < -32768)).sum())
    out["p1_near"] = int(((np.abs(p1) >= 30000) & (p1 <= 32767) & (p1 >= -32768)).sum())
    # pass-2 samples where jidctint.c's table and the saturation disagree, in DC-only blocks
    # whose pass-1 shortcut does not wrap (so pass 1 agrees)
    sel = dc_only & (np.abs(c[:, 0, 0] * q[:, 0, 0]) <= 8191)
    qs = q.reshape(-1, 64)[sel]
    cs = c.reshape(-1, 64)[sel]
    out["p2_disagree"] = sum(int((O.idct_islow(cs[i:i + 1], qs[i]) !=
                                  O.idct_islow(cs[i:i + 1], qs[i], "c")).sum())
                             for i in range(len(cs)))
    out["wrap_zero"] = int((raw_ac & ~x[:, 1:, :].any(axis=(1, 2))).sum())
    out["row0_ac"] = int((~raw_ac & c[:, 0, 1:].any(axis=1)).sum())
    for v in (32767, 32768, 65535):
        out[f"q_{v}"] = int(sum((t[2] == v).sum() for t in hd.tables))
    out["conforming_blocks"] = int((np.abs(c.reshape(-1, 64)[:, 1:]) <= 1023).all(axis=1).sum())
    out["checker_blocks"] = int((dc_only & (np.abs(c[:, 0, 0] * q[:, 0, 0]) == 1024)).sum())
    if hd.ncomp == 3 and hd.hmax > 1:
        out[f"chroma_w{-(-hd.width // hd.hmax)}"] = 1
    dcs = np.asarray(trace.get("dc", []), dtype=np.int64)
    out["dc_outside_int16"] = int(((dcs < -32768) | (dcs > 32767)).sum())
    for cat in range(12, 16):
        out[f"dc_cat_{cat}"] = trace.get("dc_cat", []).count(cat)
    for cat in range(11, 16):
        out[f"ac_cat_{cat}"] = trace.get("ac_cat", []).count(cat)
    out["ac_code_len_16"] = _has_len16(blob)
    out["eob_blocks"] = int((~c.reshape(-1, 64)[:, 1:].any(axis=1)).sum())
    out["zrl_to_63"] = trace.get("zrl_to_63", 0)
    out["run_past_63"] = trace.get("run_past_63", 0)
    scan = _scan(blob)
    out["fill_bytes"] = _fill_before_markers(blob[hd.scan_off:])
    units = [_unstuff(u) for u in _units(scan)]
    out["restart_units"] = len(units)
    for bits in {len(u) * 8 for u in units}:
        out[f"units_of_{bits}_bits"] = sum(len(u) * 8 == bits for u in units)
    flat = b"".join(units)
    for S in (32, 64, 128, 256, 512, 1024, 2048, 4096):
        out[f"ff_at_S_{S}"] = int(any(flat[p] == 0xFF for p in range(S // 8, len(flat), S // 8)))
    out["dc_pairs"] = int(dc_only.sum()) // 3 if hd.ncomp == 3 else 0
    return out


def _has_len16(blob):
    """1 when a DHT of the file assigns a code of 16 bits."""
    pos = 2
    while blob[pos + 1] != 0xDA:
        n = (blob[pos + 2] << 8) | blob[pos + 3]
        if blob[pos + 1] == 0xC4:
            seg, q = blob[pos + 4:pos + 2 + n], 0
            while q < len(seg):
                bits = seg[q + 1:q + 17]
                if bits[15]:
                    return 1
                q += 17 + sum(bits)
        pos += 2 + n
    return 0


def _fill_before_markers(scan):
    """0xFF bytes that precede another 0xFF (fill bytes before a marker)."""
    return sum(1 for i in range(len(scan) - 1) if scan[i] == 0xFF and scan[i + 1] == 0xFF)


def _units(scan):
    out, last, i = [], 0, 0
    while i < len(scan) - 1:
        if scan[i] == 0xFF and scan[i + 1] != 0x00:
            j = i
            while j < len(scan) and scan[j] == 0xFF:
                j += 1
            if j < len(scan) and 0xD0 <= scan[j] <= 0xD7:
                out.append(scan[last:i])
                last = i = j + 1
                continue
            break
        i += 2 if scan[i] == 0xFF else 1
    return out + [scan[last:].rstrip(b"\xff")]


def _unstuff(b):
    return b.replace(b"\xff\x00", b"\xff")


@pytest.mark.parametrize("builder", E.BUILDERS, ids=lambda b: b.__name__)
def test_builder_counts(builder):
    rng = np.random.default_rng(0)
    for c in builder(rng):
        got = census(c)
        for k, v in c.counts.items():
            assert got.get(k) == v, (c.name, k, got.get(k), v)
        assert any(v > 0 for v in c.counts.values()), c.name


def test_golden_is_current():
    """The committed files are the ones the builders make now."""
    g = golden()
    names = [c.name for c in cases()]
    assert list(g["names"]) == names
    for i, c in enumerate(cases()):
        assert hashlib.sha256(c.blob).hexdigest() == str(g["file_sha256"][i]), c.name


def _expected(i):
    """The golden cv2 decode of case i: the array, or (shape, sha256) for a large one; None when
    cv2 refused the file."""
    g = golden()
    name = g["names"][i]
    if not g["cv2_ok"][i]:
        return None
    if f"px_{name}" in g:
        return g[f"px_{name}"]
    return tuple(g["shape"][i]), str(g["px_sha256"][i])


def _matches(img, exp):
    if isinstance(exp, tuple):
        return img.shape == exp[0] and hashlib.sha256(img.tobytes()).hexdigest() == exp[1]
    return img.shape == exp.shape and np.array_equal(img, exp)


def test_oracle_equals_golden_cv2():
    for i, c in enumerate(cases()):
        exp = _expected(i)
        got = _oracle_of(c.name)
        if c.refused:
            assert isinstance(got, J.JpegError), c.name
            assert (exp is not None) == c.cv2_decodes, c.name
            continue
        assert exp is not None and not isinstance(got, Exception), c.name
        assert _matches(got, exp), c.name


@pytest.mark.skipif(not _is_avx2_x86(), reason="cv2's libjpeg-turbo runs its x86-64 AVX2 IDCT "
                    "only on x86-64 with AVX2; elsewhere the committed decodes stand in for it")
def test_oracle_equals_live_cv2():
    for c in cases():
        ref = JI.cv2_decode(c.blob)
        if c.refused:
            assert (ref is not None) == c.cv2_decodes, c.name
            continue
        assert np.array_equal(_oracle_of(c.name), ref), c.name


@pytest.mark.skipif(not _is_avx2_x86(), reason="the full-size colour grids are checked against "
                    "live cv2 only where it runs the x86-64 AVX2 code")
def test_full_colour_grids_equal_golden_live():
    g = golden()
    for c in E.colour_grids(step=1):
        img = JI.cv2_decode(c.blob)
        assert hashlib.sha256(img.tobytes()).hexdigest() == str(g[f"grid_sha256_{c.name}"])


@pytest.mark.parametrize("mistake", O.MISTAKES)
def test_every_idct_mistake_changes_the_expected_pixels(mistake):
    changed = []
    for c in cases():
        if c.refused or "_prog_" in c.name:
            continue
        good = _oracle_of(c.name)
        if not np.array_equal(O.decode(c.blob, mistake), good):
            changed.append(c.name)
    assert changed, mistake


def test_refusal_parity():
    """cv2 returns None exactly where jpeg.parse / Plan raises; a file the device refuses after
    the parse (a DC sum past int32) is the stated difference of DESIGN §3.20."""
    g = golden()
    for i, c in enumerate(cases()):
        try:
            J.plan_batch([c.blob])
            host_ok = True
        except J.JpegError:
            host_ok = False
        assert host_ok == bool(g["cv2_ok"][i]), c.name
        assert c.refused == (not host_ok or c.cv2_decodes), c.name
