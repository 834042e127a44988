"""Workspace sizes of the standalone conv entries (dd_conv3x3, dd_conv3x3_wgrad) for every conv shape of the DDIM loop.
They are host arithmetic, so no device is needed.  The geometries run from one 8x16 image (one weight-gradient chunk)
through an odd grid to config 3's 4 x 176 x 608 latent, where the weight gradient's split-K plan is at its widest."""
import pytest

import diffusiondepth_b200 as dd

SHAPES = [(16, 64), (64, 256), (256, 256), (256, 64), (64, 16)]  # (cin, cout)
# (batch, height, width) -> (conv3x3 bytes, wgrad bytes) per shape in SHAPES order
EXPECTED = {
    (1, 8, 16): [(123904, 157696), (1377280, 1509376), (5112832, 5244928), (1475584, 1509376), (148480, 157696)],
    (3, 37, 53): [(2334720, 5470208), (10218496, 16268288), (22793216, 28843008), (14736384, 16249856),
                  (3465216, 5466112)],
    (8, 114, 152): [(53306368, 98296832), (214107136, 381387776), (430572544, 672171008), (320570368, 380969984),
                    (79922176, 98192384)],
    (4, 176, 608): [(164439040, 283806720), (658637824, 1162355712), (1319633920, 2014454784),
                    (987366400, 1161071616), (246621184, 283486208)],
}


@pytest.mark.parametrize("geom", list(EXPECTED))
def test_standalone_conv_workspace_bytes(geom):
    lib = dd.load_library()
    b, h, w = geom
    for (cin, cout), (conv, wgrad) in zip(SHAPES, EXPECTED[geom]):
        assert lib.dd_conv3x3_workspace_bytes(b, cin, cout, h, w) == conv, (cin, cout)
        assert lib.dd_conv3x3_wgrad_workspace_bytes(b, cin, cout, h, w) == wgrad, (cin, cout)
        assert conv % 1024 == 0 and wgrad % 1024 == 0
