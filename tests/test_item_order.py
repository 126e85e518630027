"""CPU: the tile kernels' block -> item order (nsb_tile.cuh item_of_block, nsb_render.cu item_order), restated here.  Every launch must run
each (tile, decoder) item exactly once, whatever the SM count, split, batch size and resident CTAs per SM; split == 1 keeps block = tile.
A launch that is resident at once runs decoder-major, so its fine-decoder items (decoder 0) all come in the first round of blocks, where
every SM gets one block: whichever SM a later block reaches, no SM runs two fine items.  Launches of several rounds, and kernels of one CTA
per SM, stay tile-major."""
import itertools

import pytest


def item_order(tiles, split, ctas_per_sm, sms):
    return ctas_per_sm > 1 and split > 1 and tiles * split <= ctas_per_sm * sms


def item_of_block(b, n, split, kind_major):
    d = n // split if kind_major else split
    q, r = b // d, b - (b // d) * d
    return (r, q) if kind_major else (q, r)


def items(tiles, split, ctas_per_sm, sms):
    n = tiles * split
    kind_major = item_order(tiles, split, ctas_per_sm, sms)
    return [item_of_block(b, n, split, kind_major) for b in range(n)]


TILES = (1, 2, 5, 24, 43, 44, 45, 66, 67, 75, 88, 96, 131, 132, 133, 176, 263, 264, 265, 374, 375, 1000, 4096)
SMS = (1, 2, 7, 66, 78, 114, 132, 144)


@pytest.mark.parametrize("sms", SMS)
def test_every_item_once(sms):
    for tiles, split, cpb in itertools.product(TILES, (1, 2, 3), (1, 2)):
        got = items(tiles, split, cpb, sms)
        assert sorted(got) == [(t, q) for t in range(tiles) for q in range(split)], (tiles, split, cpb, sms)
        if split == 1:
            assert got == [(t, 0) for t in range(tiles)]


@pytest.mark.parametrize("sms", SMS)
def test_resident_launch_has_its_fine_items_in_the_first_round(sms):
    for tiles, split in itertools.product(TILES, (2, 3)):
        n = tiles * split
        if n > 2 * sms:
            continue
        got = items(tiles, split, 2, sms)
        assert all(q != 0 for _, q in got[sms:]), (tiles, split, sms)
        assert got[:tiles] == [(t, 0) for t in range(tiles)]


def test_headline_launch():
    """200 rays x 48 samples on 132 SMs: 75 tiles x 3 decoders, fine items in blocks 0..74, the second round colour and middle items."""
    got = items(75, 3, 2, 132)
    assert [q for _, q in got] == [0] * 75 + [1] * 75 + [2] * 75


def test_several_rounds_and_one_cta_per_sm_stay_tile_major():
    """The 996-ray mapping backward (fine + middle decoders, 374 tiles) has more items than resident slots; the weight-gradient kernels run
    one CTA per SM."""
    assert items(374, 2, 2, 132) == [(t, q) for t in range(374) for q in range(2)]
    assert items(100, 3, 1, 132) == [(t, q) for t in range(100) for q in range(3)]
