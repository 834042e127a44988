"""Pin the CPU restatement (oracle/restate.py) and the mirror's step-invariant producers against golden
vectors generated from the REAL reference (oracle/make_golden.py, oracle/make_ref_fixtures.py)."""
import pytest
import torch

from oracle import configs, restate
import dd_helpers as helpers

TOL_Z = 5e-5  # fp32-vs-fp32 re-association noise on the logits (SURVEY.md §7.2: 3e-5 vs fp64 over 20 steps)


@pytest.mark.parametrize("case", ["g_res18_c1", "g_res18_ragged", "g_mpvit_small", "g_mpvit_trained", "g_res18_trained",
                                  "g_swinl_small_trained", "g_swinl_odd_trained", "g_res18_vis_trained"])
def test_oracle_reproduces_reference_golden(case):
    """`*_trained`: the trained-like regime (oracle.configs.trainedify: random non-zero Swin relative-position tables,
    non-trivial BatchNorm running statistics, LayerNorm / GroupNorm affines) — what released checkpoints look like."""
    g = helpers.load_golden(case)
    m = helpers.build_mirror(g["family"], g["T"], helpers.is_trained_case(case))
    sd = m.state_dict()
    ck = helpers.weight_checksum(sd)
    assert abs(ck - float(g["z"]["weight_checksum"])) <= 1e-6 * ck, "weights were not regenerated identically"
    sample, noise = helpers.inputs_for(g)
    out = restate.forward(sd, sample, configs.FAMILIES[g["family"]]["backbone_name"], g["T"], noise)
    z_ref = torch.from_numpy(g["z"]["logits"])
    assert (helpers.golden_view(g, "logits", out["logits"]) - z_ref).abs().max().item() < TOL_Z
    lat_ref = torch.from_numpy(g["z"]["latent"])
    lat = helpers.golden_view(g, "latent", out["latent"])
    assert (lat - lat_ref).abs().max().item() < 1e-5 * max(1.0, float(g["z"]["latent_absmax"]))
    cond_ref = torch.from_numpy(g["z"]["cond"])
    assert (helpers.golden_view(g, "cond", out["cond"]) - cond_ref).abs().max().item() < 1e-5 * float(g["z"]["cond_absmax"])
    # depth itself, where exp(-z) is well conditioned
    pm = restate.parity_metrics(helpers.golden_view(g, "logits", out["logits"]), z_ref,
                                helpers.golden_view(g, "pred", out["pred"]), torch.from_numpy(g["z"]["pred"]))
    assert pm["max_rel_depth_wellcond"] < 1e-3
    assert sorted(str(k) for k in g["z"]["output_keys"]) == sorted([
        'aff', 'blur_depth_t', 'confidence', 'ddim_loss', 'gamma', 'gt_map_t', 'guidance', 'offset', 'pred',
        'pred_init', 'pred_inter', 'pred_uncertainty', 'weight_map'])


@pytest.mark.parametrize("case", ["g_res18_c1", "g_res18_ragged", "g_mpvit_small", "g_mpvit_trained", "g_res18_trained",
                                  "g_swinl_small_trained", "g_swinl_odd_trained"])
def test_mirror_producers_match_reference_condition(case):
    """backbone + FPN of the product mirror (torch ops, once per image) reproduce the reference's cond map."""
    g = helpers.load_golden(case)
    m = helpers.build_mirror(g["family"], g["T"], helpers.is_trained_case(case))
    sample, _ = helpers.inputs_for(g)
    with torch.no_grad():
        fp = m.depth_backbone(sample["rgb"])
        cond = m.depth_head._condition(m.depth_head._neck(fp))
        enc = m.depth_head.depth_transform.t(sample["gt"])
    ref = torch.from_numpy(g["z"]["cond"])
    assert (helpers.golden_view(g, "cond", cond) - ref).abs().max().item() < 1e-5 * float(g["z"]["cond_absmax"])
    assert enc.shape == (g["B"], 16, (g["H"] + 1) // 2, (g["W"] + 1) // 2)


def test_oracle_fp64_budget():
    """fp32 restatement vs its own fp64 evaluation: the error floor parity numbers are read against."""
    g = helpers.load_golden("g_res18_ragged")
    m = helpers.build_mirror(g["family"], g["T"])
    sd = m.state_dict()
    sample, noise = helpers.inputs_for(g)
    bb = configs.FAMILIES[g["family"]]["backbone_name"]
    o32 = restate.forward(sd, sample, bb, g["T"], noise, dtype=torch.float32)
    o64 = restate.forward(sd, sample, bb, g["T"], noise, dtype=torch.float64)
    assert (o32["logits"].double() - o64["logits"]).abs().max().item() < 1e-4


def test_denoiser_is_nonnegative_and_batch_independent():
    g = helpers.load_golden("g_res18_ragged")
    sd = helpers.build_mirror(g["family"], g["T"]).state_dict()
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(2, 16, 9, 11, generator=gen)
    cond = torch.randn(2, 256, 9, 11, generator=gen)
    e2 = restate.denoiser(sd, x, torch.tensor([10, 700]), cond, "res")
    e0 = restate.denoiser(sd, x[:1], 10, cond[:1], "res")
    assert (e2 >= 0).all()          # post-ReLU "noise" (SURVEY.md §3.2)
    assert torch.allclose(e2[:1], e0, atol=1e-6)


SWIN_HEAD_KW = dict(in_channels=[64, 128, 256, 512], inference_steps=3, num_train_timesteps=1000, depth_feature_dim=16,
                    loss_cfgs=[], init_cfg=None)


def swin_head_inputs():
    """Synthetic Swin-shaped feature maps (the slow Swin-L backbone is not needed on CPU), gt, initial noise."""
    gen = torch.Generator().manual_seed(2)
    H, W = 40, 56
    fp = [torch.randn(1, c, -(-H // s), -(-W // s), generator=gen) for c, s in ((192, 4), (384, 8), (768, 16), (1536, 32))]
    gt = torch.rand(1, 1, H, W, generator=gen) * 80
    noise = torch.randn(1, 16, H // 2, W // 2, generator=gen)
    return fp, gt, noise


def _checksum(sd):
    return sum(v.double().abs().sum().item() for v in sd.values() if v.is_floating_point())


def test_oracle_against_live_reference_swin_head():
    """Swin *head* path (HAHI neck + FPN + upsample_fuse loop + decoder) against the reference's own head on the same
    weights (the mirror's seeded initialisation) and inputs (its logits and depth stored by oracle/make_ref_fixtures.py)."""
    from diffusiondepth_b200.model.registry import HEADS
    ref = helpers.ref_fixtures()
    torch.manual_seed(11)
    head = HEADS.build(dict(type="DDIMDepthEstimate_Swin_ADDHAHI", **SWIN_HEAD_KW)).eval()
    with torch.no_grad():
        head.hahineck.level_embed.zero_()
    assert abs(_checksum(head.state_dict()) - float(ref["head_weight_checksum"])) <= 1e-6 * float(ref["head_weight_checksum"])
    sd = {"depth_head." + k: v for k, v in head.state_dict().items()}
    fp, gt, noise = swin_head_inputs()
    with torch.no_grad():
        cond = restate.fpn_condition(sd, restate.hahi_neck(sd, fp))
        lat = restate.ddim_loop(sd, cond, noise, 3, "swin")
        z = restate.decode_logits(sd, lat)
    assert (z - torch.from_numpy(ref["head_z"])).abs().max().item() < TOL_Z
    assert torch.allclose(restate.decode(sd, lat), torch.from_numpy(ref["head_pred"]), rtol=1e-4, atol=1e-6)


WMSA_C, WMSA_HEADS = 96, 3
WMSA_CASES = [((24, 40), 0), ((24, 40), 3), ((13, 9), 3)]


def wmsa_inputs(hw):
    gen = torch.Generator().manual_seed(6)
    table = torch.randn(169, WMSA_HEADS, generator=gen) * 0.7
    x = torch.randn(2, hw[0] * hw[1], WMSA_C, generator=gen)
    return table, x


@pytest.mark.parametrize("hw,shift", WMSA_CASES)
def test_window_msa_live_reference_trained_regime(hw, shift):
    """The reference's own ShiftWindowMSA / WindowMSA modules (backbone/swin.py:150-189, 250-325) with NON-ZERO
    relative-position tables, padded (24x40 -> 28x42, 13x9 -> 14x14) and shifted windows (a seeded sample of their output
    stored by oracle/make_ref_fixtures.py) against (a) the restatement and (b) the mirror's module on the same weights —
    the bias / mask / roll path that the `nopretrain` factory leaves at zero."""
    from diffusiondepth_b200.model.backbone import swin as mirror_swin
    ref = helpers.ref_fixtures()
    i = WMSA_CASES.index((hw, shift))
    torch.manual_seed(5)
    mine = mirror_swin.ShiftWindowMSA(WMSA_C, WMSA_HEADS, 7, shift).eval()
    assert abs(_checksum(mine.state_dict()) - float(ref[f"wmsa_{i}_weight_checksum"])) <= 1e-6 * float(ref[f"wmsa_{i}_weight_checksum"])
    table, x = wmsa_inputs(hw)
    with torch.no_grad():
        mine.w_msa.relative_position_bias_table.copy_(table)
    idx = torch.from_numpy(helpers.fixture_sample_index(2 * hw[0] * hw[1] * WMSA_C))
    want = torch.from_numpy(ref[f"wmsa_{i}_sample"])
    tol = 2e-6 * float(ref[f"wmsa_{i}_absmax"]) + 1e-6
    sd = {"a." + k: v for k, v in mine.state_dict().items()}
    got = restate._shift_window_msa(sd, x, hw, "a.", WMSA_HEADS, 7, shift)
    assert (got.reshape(-1)[idx] - want).abs().max().item() < tol
    with torch.no_grad():
        assert (mine(x, hw).reshape(-1)[idx] - want).abs().max().item() < tol
    # the bias really matters in this regime
    sd["a.w_msa.relative_position_bias_table"] = torch.zeros_like(table)
    nobias = restate._shift_window_msa(sd, x, hw, "a.", WMSA_HEADS, 7, shift)
    assert (nobias.reshape(-1)[idx] - want).abs().max().item() > 1e-3
