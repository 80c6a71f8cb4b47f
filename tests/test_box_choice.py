"""Output-box choice of the GEMM engine (ops.pick_box, also used by the FGT model): fewest 128-row tiles."""
from fgt_b200 import ops


def _tiles(box, ow, oh):
    return -(-ow // box[0]) * -(-oh // box[1])


def test_boxes_fit_the_engine():
    assert len(set(ops._BOXES)) == len(ops._BOXES)
    for bw, bh in ops._BOXES:
        assert bw * bh <= 128 and bw * bh % 8 == 0


def test_token_grid_box():
    # patch2vec / f_patch2vec output grid (432x240 input): 36 x 20 tokens, 720 positions in 6 tiles of 120
    assert ops.pick_box(36, 20) == (12, 10)
    assert _tiles(ops.pick_box(36, 20), 36, 20) == 6


def test_fewest_tiles_and_ties_keep_the_old_boxes():
    old = ((16, 8), (32, 4), (8, 16), (64, 2), (128, 1))
    for ow, oh in ((432, 240), (216, 120), (108, 60), (54, 30), (36, 20), (27, 15), (333, 1), (7, 3), (1, 1)):
        box = ops.pick_box(ow, oh)
        best = min(_tiles(b, ow, oh) for b in ops._BOXES)
        assert _tiles(box, ow, oh) == best
        best_old = min(old, key=lambda b: _tiles(b, ow, oh))
        if _tiles(best_old, ow, oh) == best:
            assert box == best_old, (ow, oh, box)
