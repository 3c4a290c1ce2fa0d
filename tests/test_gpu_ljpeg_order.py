"""k2_stream_kernel decodes the thread path's segments in the plan's order (thread_shape_order in
rawspeed_b200/csrc/ljpeg_host.h: by tile shape, not by scan order), so everything indexed by a thread's
position -- the redo flags the tile kernel's second opinion reads among them -- must follow that order.
A batch of tiled frames with one, two and four components, each with interior, right-edge, bottom and
corner tiles, some segments truncated (the tile kernel's redo) and some with an unassigned code
(status 1), in both forms of the kernel: the whole output buffer, and (status, consumed) of every
segment, against the oracle."""
import numpy as np
import pytest

import rawspeed_b200 as rs
from oracle import port, synth
from helpers import dng_ljpeg_scans
from test_gpu_ljpeg import set_ljpeg_path
from test_gpu_ljpeg_edges import _huffs, _oracle, _run

pytestmark = pytest.mark.gpu

W, H, TW, TH = 1000, 100, 128, 16   # 8 x 7 tiles: the last column 104 samples wide, the last row 4 high
CUTS = (1, 3, 8, 17)


def _batch():
    """Two frames per component count, stacked in one output buffer; in every frame some tiles of each
    shape truncated by CUTS bytes and some given an unassigned code.  Returns (tables, scans, input,
    output shape, expected output, expected (status, consumed) per scan)."""
    pitch = port.image_pitch(W)
    tabs, scans, blobs = None, [], []
    base = 0
    for f, g in enumerate((1, 1, 2, 2, 4, 4)):
        img = synth.image_model(W, H, 100 + f, wild=f % 2 == 1)
        t = synth.make_dng_ljpeg(img, TW, TH, ncomp=g)
        tabs, sc = dng_ljpeg_scans(t, pitch, out_offset=f * H * pitch, in_base=base, tabs=tabs)
        blob = t.blob.copy()
        for k, s in enumerate(sc):
            if (k + f) % 5 == 2:                        # truncated
                s.in_size -= CUTS[(k + f) % len(CUTS)]
            elif (k + f) % 9 == 4:                      # an unassigned code: 39 one-bits at byte 40
                o = s.in_offset - base
                pos = o + (41 if blob[o + 39] == 0xFF else 40)
                blob[pos:pos + 9] = [0xFF, 0, 0xFF, 0, 0xFF, 0, 0xFF, 0, 0xFE]
        scans += sc
        blobs.append(blob)
        base += blob.size
    data = np.concatenate(blobs)
    want = port.new_image(W, H * 6)
    huffs = _huffs(tabs)
    wants = [_oracle(s, data[s.in_offset:s.in_offset + s.in_size], huffs,
                     want[s.out_offset // pitch:s.out_offset // pitch + H]) for s in scans]
    return tabs, scans, data, want, wants


@pytest.mark.parametrize("form", ["prefetch", "wide"])
def test_shape_order_with_redo_and_bad_codes(ctx, monkeypatch, form):
    tabs, scans, data, want, wants = _batch()
    st = [w[0] for w in wants]
    assert st.count(1) >= 6 and st.count(2) >= 6
    shapes = {(s.mcu_w, s.store_w, s.rows) for s in scans}
    assert len(shapes) == 12                             # 3 component counts x 4 tile shapes
    set_ljpeg_path(monkeypatch, "stream")
    monkeypatch.setenv("RSB200_STREAM_FORM", form)
    plan = rs.ljpeg_plan(ctx, tabs.tabs, scans)
    kinds = plan.kernels
    assert ("full-launch form" if form == "wide" else "prefetch form") in kinds, kinds
    assert "k2_tile_kernel<1> for flagged ends of stream" in kinds, kinds
    got, res = _run(plan, data, port.new_image(W, H * 6))
    # (status, consumed) of every segment; the whole buffer, but for the rows of segments that failed
    pitch = port.image_pitch(W)
    got, want = got.copy(), want.copy()
    for k, (s, (ws, wc), (gs, gc)) in enumerate(zip(scans, wants, res)):
        assert gs == ws, (k, gs, ws)
        if ws == 0:
            assert gc == wc, (k, gc, wc)
        else:
            y = s.out_offset // pitch + s.out_y
            got[y:y + s.rows, s.out_x:s.out_x + s.store_w] = 0
            want[y:y + s.rows, s.out_x:s.out_x + s.store_w] = 0
    bad = np.argwhere(got != want)
    assert bad.size == 0, (bad[:5], got[tuple(bad[0])], want[tuple(bad[0])])
