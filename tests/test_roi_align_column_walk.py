"""CPU model of the column-shared bin walk of roi_align_nhwc_kernel (detectron2_b200/csrc/roi_align.cu: the owned-column table
built by warp 1 and nhwc_unit): the table rules and the two-accumulator walk, restated in Python on one channel, against the
direct double sum over the per-bin tap lists.  Documents WHY the walk is exact: a column belongs to the first bin that touches
it (weight wa) and may reach the next bin (weight wb); a column that touches three bins disqualifies the RoI (per-bin loop);
a bin without an owned column still gets one zero-weight entry so that every bin ends on a flagged entry.  The GPU tests
(tests/test_gpu_parity.py) check the kernel itself against the oracle."""
import math

import numpy as np
import pytest


def make_tap1(v, size):  # roi_align.cu make_tap1 / torchvision bilinear_interpolate, one axis
    if v < -1.0 or v > size:
        return 0, 0, 0.0, 0.0
    v = max(v, 0.0)
    lo = int(v)
    if lo >= size - 1:
        hi = lo = size - 1
        v = float(lo)
    else:
        hi = lo + 1
    frac = v - lo
    return lo, hi, 1.0 - frac, frac


def sample_pos(start, bin_size, grid, p, i, fp32=False):
    """Position of sample i of bin p along one axis; fp32: as the kernels compute it (start, bin_size fp32 values from
    load_geom), start + p*bin + ((i + .5)*bin)/grid rounded after every operation."""
    if not fp32:
        return start + p * bin_size + (i + 0.5) * bin_size / grid
    f = np.float32
    s, b = f(start), f(bin_size)
    return float((s + f(p) * b) + (f(i) + f(0.5)) * b / f(grid))


def tap_list(start, bin_size, grid, p, size, fp32=False):
    """add_tap: the (index, weight) list of bin p along one axis, samples merged per index.  fp32: sample positions in fp32
    (sample_pos), weights and their sums in float64."""
    lst = []
    for i in range(grid):
        lo, hi, wl, wh = make_tap1(sample_pos(start, bin_size, grid, p, i, fp32), size)
        for idx, w in ((lo, wl), (hi, wh)):
            if w == 0:
                continue
            for e in lst:
                if e[0] == idx:
                    e[1] += w
                    break
            else:
                lst.append([idx, w])
    return lst


def owned_columns(xlists):
    """The table warp 1 builds: entries [column, wa, wb, last-of-bin flag] bin after bin, cbeg; None if a column touches three
    consecutive bins (the kernel then takes the per-bin loop)."""
    pw = len(xlists)
    entries, cbeg = [], [0] * (pw + 1)
    for b in range(pw):
        prev1 = xlists[b - 1] if b >= 1 else []
        prev2 = xlists[b - 2] if b >= 2 else []
        nxt = xlists[b + 1] if b + 1 < pw else []
        own = []
        for c, w in xlists[b]:
            in1 = any(q[0] == c for q in prev1)
            if in1 and any(q[0] == c for q in prev2):
                return None, None
            if not in1:
                own.append((c, w))
        cbeg[b] = len(entries)
        for i, (c, w) in enumerate(own):
            wb = next((q[1] for q in nxt if q[0] == c), 0.0)
            entries.append([c, w, wb, 1 if i == len(own) - 1 else 0])
        if not own:
            entries.append([0, 0.0, 0.0, 1])
    cbeg[pw] = len(entries)
    entries += [[0, 0.0, 0.0, 0]] * 4  # chunk padding read (and masked) by the XC-wide loop
    return entries, cbeg


def walk(feat, ylists, entries, cbeg, ph_count, pw_count, count):
    """nhwc_unit over every unit of 7 bins: rotating accumulators (cur, nxt), emission at flagged entries, carry-in bin for
    units that do not start a row, tap rows in chunks of <= 6 with accumulation into the output on later chunks."""
    xc_of = {1: 4, 2: 3, 3: 2, 4: 1, 5: 1, 6: 1}
    out = np.full((ph_count, pw_count), np.nan)
    for u in range(ph_count * pw_count // 7):
        fb = u * 7
        ph, pw0 = fb // pw_count, fb % pw_count
        rows = ylists[ph]
        if not rows:
            out[ph, pw0:pw0 + 7] = 0.0
            continue
        skip = 1 if pw0 > 0 else 0
        cb, ce = cbeg[pw0 - skip], cbeg[pw0 + 7]
        nch = (len(rows) + 5) // 6
        ry = (len(rows) + nch - 1) // nch
        xc = xc_of[ry]
        for ch in range(nch):
            chunk = [(rows[e][0], rows[e][1]) if e < len(rows) else (rows[0][0], 0.0) for e in range(ch * ry, ch * ry + ry)]
            cur = nxt = 0.0
            b = -skip
            for s in range(cb, ce, xc):
                for x in range(xc):
                    col, wa, wb, flag = entries[s + x]
                    live = xc == 1 or s + x < ce
                    t = sum(wy * feat[y, col] for y, wy in chunk)
                    cur += (wa if live else 0.0) * t
                    nxt += (wb if live else 0.0) * t
                    if live and flag:
                        if b >= 0:
                            out[ph, pw0 + b] = cur / count if ch == 0 else out[ph, pw0 + b] + cur / count
                        cur, nxt, b = nxt, 0.0, b + 1
    return out


def test_column_walk_equals_per_bin_double_sum():
    rng = np.random.default_rng(0)
    checked = fallback = 0
    for _ in range(500):
        h, w = int(rng.integers(6, 60)), int(rng.integers(6, 60))
        feat = rng.standard_normal((h, w))
        pw_count = int(rng.choice([7, 14]))
        ph_count = int(rng.choice([7, 14, 5, 3]))
        scale = float(rng.choice([0.3, 1, 2, 4, 8]))
        x1, y1 = rng.uniform(-5, w), rng.uniform(-5, h)  # partly outside the map: clamped / dropped samples
        bw, bh = rng.uniform(0.5, 10) * scale, rng.uniform(0.5, 10) * scale
        sr = int(rng.choice([0, 0, 0, 2, 1]))
        gh = sr if sr > 0 else int(math.ceil(bh / ph_count))
        gw = sr if sr > 0 else int(math.ceil(bw / pw_count))
        if gh > 16 or gw > 16:
            continue
        count = max(gh * gw, 1)
        ylists = [tap_list(y1 - 0.5, bh / ph_count, gh, p, h) for p in range(ph_count)]
        xlists = [tap_list(x1 - 0.5, bw / pw_count, gw, p, w) for p in range(pw_count)]
        ref = np.array([[sum(wy * wx * feat[y, x] for y, wy in yl for x, wx in xl) / count for xl in xlists] for yl in ylists])
        entries, cbeg = owned_columns(xlists)
        if entries is None:
            fallback += 1
            continue
        got = walk(feat, ylists, entries, cbeg, ph_count, pw_count, count)
        assert not np.isnan(got).any()
        assert np.abs(got - ref).max() < 1e-9
        assert all(cbeg[b + 1] > cbeg[b] for b in range(pw_count))  # every bin owns at least one (possibly dummy) entry
        checked += 1
    assert checked > 150 and fallback > 50  # both outcomes of the three-bin test occur


def test_three_bins_on_one_column_disqualify_the_walk():
    # bins narrower than a pixel: one column is touched by three consecutive bins
    xlists = [tap_list(10.0, 0.4, 1, p, 64) for p in range(7)]
    assert owned_columns(xlists) == (None, None)
    # bins two pixels wide: every column touches at most two bins
    xlists = [tap_list(10.3, 2.0, 2, p, 64) for p in range(7)]
    entries, cbeg = owned_columns(xlists)
    assert entries is not None and cbeg[7] <= sum(len(x) for x in xlists)
