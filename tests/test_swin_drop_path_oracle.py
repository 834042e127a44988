"""Swin-L's stochastic depth in the mirror and in the head's draw helper, on the CPU, against the real reference in
`.train()` (tests/golden/g_swin_drop_path.npz, oracle/make_swin_drop_path.py): the same schedule, the same mmcv DropPath
draws from the same seeded generator, the same stage features and the same generator state after the forward.  Also
the layout the head hands the engine, and that the mirror's factories keep stochastic depth off."""
import copy

import numpy as np
import pytest
import torch

import dd_helpers as helpers
from diffusiondepth_b200.model._blocks import MMCVDropPath
from oracle.make_denoiser_grads import checksum, sample_index
from oracle.make_swin_drop_path import B, CASES, FAMILY, OUT, RATE, case_rgb, case_seed


@pytest.fixture(scope="module")
def golden():
    return np.load(OUT, allow_pickle=False)


def mirror_swin(rate):
    """The trained-like mirror Swin-L in training mode at drop-path rate `rate`, fp32 on the CPU."""
    bb = copy.deepcopy(helpers.build_mirror(FAMILY, 2, trained=True).depth_backbone).train()
    bb.set_drop_path_rate(rate)
    return bb


def _rates(bb):
    return [(blk.attn.drop.drop_prob, blk.ffn.dropout_layer.drop_prob) for st in bb.stages for blk in st.blocks]


def test_factories_keep_stochastic_depth_off():
    model = helpers.build_mirror(FAMILY, 2)
    bb, head = model.depth_backbone, model.depth_head
    assert all(r == (0.0, 0.0) for r in _rates(bb))
    assert head.swin_drop_paths(bb) == ((0, 0, 0, 0), [])
    assert head._native_drop_paths((64, 96), bb) is None  # the engine key and the engine stay as they were
    fresh = copy.deepcopy(bb)
    fresh.set_drop_path_rate(0.1)
    assert list(fresh.state_dict()) == list(bb.state_dict())  # no new parameters or buffers


def test_schedule_and_layout():
    """linspace(0, rate, 24) over the blocks in order (the reference's running slice of dpr), both branches of a block
    at its rate, and the head's marks / draw order."""
    bb = mirror_swin(0.1)
    rates = torch.linspace(0, 0.1, 24)
    assert _rates(bb) == [(r.item(), r.item()) for r in rates]
    head = helpers.build_mirror(FAMILY, 2).depth_head
    masks, mods = head.swin_drop_paths(bb)
    assert masks == (0b10, 0b11, (1 << 18) - 1, 0b11) and len(mods) == 2 * 23
    blocks = [blk for st in bb.stages for blk in st.blocks][1:]
    assert all(m is x for m, x in zip(mods, [d for blk in blocks for d in (blk.attn.drop, blk.ffn.dropout_layer)]))
    assert head._native_drop_paths((64, 96), bb)[0] == masks
    bb.eval()
    assert head._swin_drop_scales(bb, 2, "cpu") is None  # nothing in training mode: nothing drawn
    one = bb.stages[2].blocks[5].ffn.dropout_layer.train()
    i = next(k for k, m in enumerate(mods) if m is one)
    torch.manual_seed(3)
    scales = head._swin_drop_scales(bb, 2, "cpu").reshape(-1, 2)
    torch.manual_seed(3)
    keep = 1.0 - one.drop_prob
    assert torch.equal(scales[i], (keep + torch.rand((2, 1, 1))).floor().reshape(2) / keep)  # the one branch that draws
    assert scales.shape == (46, 2) and bool((torch.cat([scales[:i], scales[i + 1:]]) == 1).all())


def test_mmcv_drop_path_formula():
    m = MMCVDropPath(0.25).train()
    x = torch.randn(5, 7, 3)
    torch.manual_seed(11)
    y = m(x)
    torch.manual_seed(11)
    r = (0.75 + torch.rand((5, 1, 1))).floor()
    assert torch.equal(y, x.div(0.75) * r)
    m.eval()
    g = torch.get_rng_state()
    assert m(x) is x and torch.equal(g, torch.get_rng_state())


@pytest.mark.parametrize("case", list(CASES))
def test_mirror_matches_reference_train(case, golden):
    rgb = case_rgb(case)
    assert checksum(rgb) == pytest.approx(float(golden[case + "/input_checksum"]), rel=1e-12)
    bb = mirror_swin(RATE)
    sd = {k: v for k, v in bb.state_dict().items() if v.is_floating_point() and "relative_position_index" not in k}
    assert checksum(*sd.values()) == pytest.approx(float(golden[case + "/weight_checksum"]), rel=1e-9)
    torch.manual_seed(case_seed(case))
    with torch.no_grad():
        feats = bb(rgb)
    assert torch.equal(torch.get_rng_state(), torch.from_numpy(golden[case + "/rng_state"]))
    worst = 0.0
    for i, f in enumerate(feats):
        flat = f.reshape(-1)
        ref = torch.from_numpy(golden[f"{case}/feats/{i}/values"])
        got = flat[torch.from_numpy(sample_index(flat.numel()))]
        worst = max(worst, ((got.double() - ref.double()).abs().max() / float(golden[f"{case}/feats/{i}/absmax"])).item())
    print(f"\n[{case}] fp32 mirror vs fp32 reference at drop_path_rate {RATE}: feats {worst:.1e}")
    assert worst <= 2e-6


@pytest.mark.parametrize("case", list(CASES))
def test_head_draw_reproduces_reference_masks(case, golden):
    """The head's draw helper, from the same seed, draws the reference's masks and leaves the generator where the
    reference's forward left it (nothing else in the reference's Swin draws)."""
    bb = mirror_swin(RATE)
    head = helpers.build_mirror(FAMILY, 2).depth_head
    torch.manual_seed(case_seed(case))
    scales = head._swin_drop_scales(bb, B, "cpu").reshape(-1, B)
    masks = golden[case + "/masks"]
    assert torch.equal((scales > 0).to(torch.uint8), torch.from_numpy(masks))
    assert torch.equal(torch.get_rng_state(), torch.from_numpy(golden[case + "/rng_state"]))
    keep = torch.tensor([1.0 - m.drop_prob for m in head.swin_drop_paths(bb)[1]])
    assert torch.equal(scales, torch.from_numpy(masks).float() / keep[:, None])
    assert 0 < masks[4:40].sum() < masks[4:40].size  # stage 2: some images dropped, some kept
