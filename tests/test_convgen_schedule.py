"""convgen_wgmma_kernel's schedule against fp64 at the work counts where it can go wrong.  The kernel cuts each CTA's
work items into units (128 rows x NT / 2 columns for NT = 192 / 256, the whole item for NT = 64 / 128) that its two
consumer warpgroups take in turn, while the producers stream the units' K chunks through one stage ring.  The cases
below pin a CTA with a single work item, a CTA with one item more than the others, warpgroups of one CTA with unequal
unit counts, alternating whole items, a layer split along K, and K = 64, where every unit is one stage and the ring
wraps across units and warpgroups.  Each case goes through dd_gen_layer, is held to the bound of
test_producer_layers.py and repeats bit-identically."""
import pytest

from test_producer_layers import DEV, Case, _check, _sms

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import diffusiondepth_b200 as dd
    e = dd.DenoiseEngine("swin", 1, (8, 16), (4, 8), 2, DEV, cuda_graph=False)
    yield e
    e.close()


def _run(case, eng):
    return _check(case, eng, case.c0 * 13 + case.cout, {})


@gpu
@pytest.mark.parametrize("nt", [256, 192])
def test_single_work_item(eng, nt):
    """One 128 x NT item: grid 1, each warpgroup takes one of its two units."""
    info = _run(Case(f"one.item.nt{nt}", 192, nt, M=100, bias=True, add="after", n_tile=nt, alt_tile=-1,
                     regimes=("signed", "relu")), eng)
    assert info["nt"] == nt and info["work"] == 1 and info["grid"] == 1, info


@gpu
@pytest.mark.parametrize("nt", [256, 192, 128, 64])
def test_work_is_grid_plus_one(eng, nt):
    """work = grid + 1: CTA 0 takes a second item, every other CTA one; at NT <= 128 CTA 0's warpgroups take one
    item each and every other CTA's second warpgroup none."""
    sms = _sms()
    info = _run(Case(f"grid+1.nt{nt}", 384, nt, M=128 * sms + 40, bias=True, act=2, out="both", n_tile=nt,
                     alt_tile=-1, regimes=("signed",)), eng)
    assert info["nt"] == nt and info["work"] == info["grid"] + 1 and info["grid"] == sms, info


@gpu
@pytest.mark.parametrize("nt", [128, 64])
def test_whole_items_alternate(eng, nt):
    """2 x grid + 3 items of NT <= 128 columns: CTAs 0-2 take three, so their first warpgroup takes two items and
    the second one; the rest take two, one per warpgroup."""
    sms = _sms()
    info = _run(Case(f"alternate.nt{nt}", 256, nt, M=128 * (2 * sms + 3), bias=True, add="after", n_tile=nt,
                     alt_tile=-1, regimes=("signed", "relu")), eng)
    assert info["nt"] == nt and info["work"] == 2 * info["grid"] + 3, info


@gpu
@pytest.mark.parametrize("nt", [256, 192])
def test_split_k(eng, nt):
    """(1536 + 512) channels x 9 taps = 288 K iterations: three launches pass partial sums through the fp32 partial
    buffer, each with more items than CTAs."""
    info = _run(Case(f"split.nt{nt}", 1536, 768, c1=512, B=2, H=48, W=64, k=3, bn=True, act=1, out="both",
                     n_tile=nt, alt_tile=-1, regimes=("signed",)), eng)
    assert info["nt"] == nt and info["parts"] == 3 and info["work"] > info["grid"], info


@gpu
@pytest.mark.parametrize("nt", [256, 192, 128, 64])
def test_k64_single_stage_units(eng, nt):
    """K = 64: one stage per unit, so consecutive units (and warpgroups) follow each other round the ring."""
    sms = _sms()
    info = _run(Case(f"k64.nt{nt}", 64, 2 * nt, M=128 * (3 * sms) + 5, bias=True, add="after", n_tile=nt,
                     alt_tile=-1, regimes=("signed", "relu")), eng)
    assert info["nt"] == nt and info["work"] > 5 * info["grid"], info

