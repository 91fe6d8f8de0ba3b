"""GPU: the CFG-split DiT forward (DiffusionTransformer.shard_tokens with two rows, satb_dit_group_create_cfg).

Row 0 runs the conditional rows of every CFG call and row 1 the unconditional rows, each row token-sharded over its own
ranks; row 0 combines the halves.  On one device the ranks are virtual (a handle and a stream each on cuda:0), which runs
the same split, gathers, combine and event schedule as ranks on distinct GPUs; those add only the peer-to-peer reads,
tested at the end when enough devices are visible.  For rows of 1, 2, 3 and 4 ranks, every case of the token-sharded
tests, and (rows of one rank only) conformer blocks, a use_conv feed-forward and FP8 self-attention:
  * the split output is within 1.25x of the operand-rounding floor of the fp32 oracle;
  * it matches the unsharded native forward within rel-L2 4e-3; whether it is bit-identical is reported, not required
    (each half runs B rows instead of 2 B, and the attention route depends on the work-unit count);
  * a repeated call, the graph replay and its replay equal the eager split call exactly;
  * a call without CFG equals shard_tokens(row 0) exactly, and shard_tokens(None) gives the unsharded result again.
`CFGSPLIT {...}` lines (pytest -s) record the errors, the bit identity and the graph counters."""
import json

import pytest
import torch

from fp8_attn_ref import fp8_attention
from helpers import SAO_DIT, build_native_dit, rel_l2
from test_gpu_dit_group import CASES, SMALL, _cuda, _floor_ctx, _inputs

pytestmark = pytest.mark.gpu

# the options a row of several ranks refuses: run at rows of one rank
ROW1_CASES = {
    "conformer": (dict(SMALL, conformer=True), "fp16", dict(cfg_scale=7.0)),
    "use_conv": (dict(SMALL, ff_kwargs=dict(glu=False, use_conv=True, conv_kernel_size=3)), "fp16", dict(cfg_scale=7.0)),
    "attention_fp8": (dict(SMALL, attention_dtype="fp8"), "fp16", dict(cfg_scale=7.0)),
}
ALL_CASES = dict(CASES, **ROW1_CASES)
PARAMS = [(case, row, L) for case in sorted(ALL_CASES) for row in (1, 2, 3, 4) for L in (300, 1100)
          if case in CASES or row == 1]


def report(**kw):
    print("CFGSPLIT", json.dumps(kw))


def _oracle_module(case):
    from oracle import conformer_oracle as co
    from oracle import dit_oracle as do
    from oracle import feedforward_oracle as fo
    from oracle import positions_oracle as po
    return {"conformer": co, "use_conv": fo, "attention_fp8": do}.get(case, po)


_ORACLE = {}


def _oracle(case, L):
    """Weights, inputs, the fp32 oracle's output and the operand-rounding floor of one case (shared by the layouts).
    FP8 self-attention's floor also rounds the attention operands as the native kernels do."""
    if (case, L) not in _ORACLE:
        cfg, dtype, extra = ALL_CASES[case]
        orc = _oracle_module(case)
        ocfg = {k: v for k, v in cfg.items() if k != "attention_dtype"}
        sd = orc.make_dit_weights(ocfg, seed=91)
        kw = _inputs(cfg, extra, L, seed=92 + L)
        ref = orc.dit_forward(sd, ocfg, **kw)
        with _floor_ctx(dtype)(sd):
            if case == "attention_fp8":
                with fp8_attention():
                    floor = rel_l2(orc.dit_forward(sd, ocfg, **kw), ref)
            else:
                floor = rel_l2(orc.dit_forward(sd, ocfg, **kw), ref)
        _ORACLE[(case, L)] = (sd, kw, ref, floor)
    return _ORACLE[(case, L)]


def _call(m, kw, graph):
    m.cuda_graph = graph
    try:
        return m(**kw).clone()
    finally:
        m.cuda_graph = False


def _rows(n):
    return [["cuda:0"] * n, ["cuda:0"] * n]


@pytest.mark.parametrize("case,row,L", PARAMS)
def test_cfg_split_vs_oracle_unsharded_graph_and_row_0(case, row, L):
    cfg, dtype, extra = ALL_CASES[case]
    sd, kw, ref, floor = _oracle(case, L)
    m = build_native_dit(cfg, sd, operand_dtype=dtype)
    kw = _cuda(kw)
    kw_plain = dict(kw, cfg_scale=1.0)                       # the same call without CFG
    y1 = _call(m, kw, False)
    y1_plain = _call(m, kw_plain, False)
    m.shard_tokens(_rows(row))
    ys = _call(m, kw, False)
    ys2 = _call(m, kw, False)                                # the group's workspaces and conditioning reused
    yg = _call(m, kw, True)                                  # warm-up, capture, first launch
    yg2 = _call(m, kw, True)                                 # a plain replay
    stats = m.shard_graph_stats()
    ys_plain = _call(m, kw_plain, False)                     # no CFG: row 0 only
    if case in CASES:
        m.shard_tokens(["cuda:0"] * row)
        yrow0_plain = _call(m, kw_plain, False)
    else:                                                    # shard_tokens(row 0) refuses these options
        yrow0_plain = None
    m.shard_tokens(None)
    y1b = _call(m, kw, False)                                # and the single-device path is as before
    ys, ys2, yg, yg2, y1, y1b = (v.cpu() for v in (ys, ys2, yg, yg2, y1, y1b))
    err_s, err_1, vs_1 = rel_l2(ys, ref), rel_l2(y1, ref), rel_l2(ys, y1)
    calls = 2 if (cfg.get("patch_size", 1) > 1 and extra.get("scale_phi", 0.0) != 0.0) else 1
    report(case=case, layout=f"{row}x2", L=L, rel_l2_split=err_s, rel_l2_unsharded=err_1, floor=floor,
           split_vs_unsharded=vs_1, bit_identical=bool(torch.equal(ys, y1)), graph_stats=stats,
           no_cfg_vs_unsharded=rel_l2(ys_plain.cpu(), y1_plain.cpu()),
           no_cfg_bit_identical_to_unsharded=bool(torch.equal(ys_plain, y1_plain)))
    assert torch.equal(ys, ys2) and torch.equal(y1, y1b)
    assert torch.equal(yg, ys) and torch.equal(yg2, ys)
    assert stats[1] == 2 * calls and stats[2] > 0
    if calls == 1:
        assert stats[0] == 1
    if yrow0_plain is not None:
        assert torch.equal(ys_plain, yrow0_plain)
    assert rel_l2(ys_plain.cpu(), y1_plain.cpu()) < 4e-3
    assert err_s <= 1.25 * floor, (err_s, floor)
    assert vs_1 < 4e-3, vs_1


def test_cfg_split_replay_with_new_inputs_equals_eager():
    cfg, dtype, extra = CASES["prepend_cfg"]
    sd, kw, ref, floor = _oracle("prepend_cfg", 1100)
    m = build_native_dit(cfg, sd, operand_dtype=dtype).shard_tokens(_rows(3))
    kw = _cuda(kw)
    _call(m, kw, True)
    g = torch.Generator().manual_seed(7)
    for i in range(3):
        kw2 = dict(kw, x=torch.randn(kw["x"].shape, generator=g).cuda(), t=torch.tensor([0.1 + 0.3 * i]).cuda())
        yg = _call(m, kw2, True)
        ye = _call(m, kw2, False)
        assert torch.equal(yg, ye)
    assert m.shard_graph_stats()[0] == 1      # new inputs in the same static buffers: no recapture


def test_cfg_split_every_key_and_state_change_recaptures_and_stays_exact():
    """cfg_scale, scale_phi, B, L, the conditioning tensors, a switch to no CFG and back, load_state_dict, another
    layout and eager calls in between: each graph result equals the eager CFG-split result for the same call."""
    cfg, dtype, extra = CASES["prepend_cfg"]
    sd, kw, ref, floor = _oracle("prepend_cfg", 300)
    m = build_native_dit(cfg, sd, operand_dtype=dtype).shard_tokens(_rows(2))
    kw = _cuda(kw)
    log = []

    def check(name, kw_, recapture=True, new_group=False):
        before = m.shard_graph_stats()
        yg = _call(m, kw_, True)
        after = m.shard_graph_stats()
        ye = _call(m, kw_, False)
        log.append(dict(step=name, stats=after, equal=bool(torch.equal(yg, ye))))
        assert torch.equal(yg, ye), name
        if new_group:
            assert after[:2] == (1, 1), (name, before, after)
        elif recapture:
            assert before is None or after[0] == before[0] + 1, (name, before, after)
        else:
            assert after[0] == before[0], (name, before, after)
        return yg

    check("first", kw)
    check("same", kw, recapture=False)
    check("cfg_scale", dict(kw, cfg_scale=3.0))
    check("scale_phi", dict(kw, cfg_scale=3.0, scale_phi=0.5))
    g = torch.Generator().manual_seed(8)
    kw_b = dict(kw, x=torch.randn(2, 64, 300, generator=g).cuda(), t=torch.tensor([0.2, 0.7]).cuda(),
                cross_attn_cond=torch.randn(2, 19, 128, generator=g).cuda(),
                global_embed=torch.randn(2, 256, generator=g).cuda())
    check("B", kw_b)
    check("L", dict(kw, x=torch.randn(1, 64, 700, generator=g).cuda()))
    check("cond", dict(kw, cross_attn_cond=torch.randn_like(kw["cross_attn_cond"])))
    check("cond_in_place", kw)
    kw["global_embed"].mul_(0.5)              # same tensor, new version: the conditioning is prepared again
    check("cond_mutated", kw)
    check("negative_prompt", dict(kw, negative_cross_attn_cond=torch.randn_like(kw["cross_attn_cond"])))
    check("no_cfg", dict(kw, cfg_scale=1.0))  # row 0 only
    check("cfg_again", kw)
    m.load_state_dict({k: v * 1.01 if v.dtype.is_floating_point else v for k, v in sd.items()})
    check("load_state_dict", kw, new_group=True)
    m.shard_tokens(_rows(3))
    check("shard_tokens", kw, new_group=True)
    yg = _call(m, kw, True)
    _call(m, dict(kw, x=torch.randn_like(kw["x"])), False)  # an eager call between two replays
    assert torch.equal(_call(m, kw, True), yg)
    _call(m, dict(kw, x=torch.randn(1, 64, 500, generator=g).cuda()), False)  # one that reserves another shape
    check("eager_reserve", kw)
    _call(m, dict(kw, cfg_scale=1.0), False)  # an eager call on row 0 only
    check("eager_no_cfg", kw)
    report(case="recapture", log=log)


def test_cfg_split_generate_diffusion_cond_graph_equals_eager_split_and_unsharded():
    """dpmpp-3m-sde, CFG 5, 6 steps and the VAE decode, with a [[0, 0], [0, 0]] DiT: the sampler's graph calls give the
    eager CFG-split run bit for bit, and the unsharded run within the bound."""
    from stable_audio_tools.inference.generation import generate_diffusion_cond
    from test_gpu_generate import _build
    model = _build()[0]
    dit = model.model.model
    B, L, steps = 2, 300, 6
    g = torch.Generator().manual_seed(96)
    cond = {"prompt": (torch.randn(B, 10, 128, generator=g).cuda(), torch.ones(B, 10).cuda()),
            "seconds_start": (torch.randn(B, 1, 128, generator=g).cuda(), torch.ones(B, 1).cuda()),
            "seconds_total": (torch.randn(B, 1, 128, generator=g).cuda(), torch.ones(B, 1).cuda())}
    sde_noise = [torch.randn(B, 64, L, generator=g).cuda() for _ in range(steps)]

    def run():
        it = iter(sde_noise)
        lat = generate_diffusion_cond(model, steps=steps, cfg_scale=5.0, conditioning_tensors=cond, sample_size=L * 64,
                                      seed=97, device="cuda", return_latents=True, sampler_type="dpmpp-3m-sde",
                                      sigma_min=0.3, sigma_max=50.0, noise_sampler=lambda s, sn: next(it))
        return lat.cpu(), model.pretransform.decode(lat).cpu()

    lat1, audio1 = run()
    dit.shard_tokens(_rows(2))
    latg, audiog = run()
    stats = dit.shard_graph_stats()
    dit.__dict__["_sharded_graph_forward"] = dit._sharded_forward    # the same run with every split call eager
    try:
        late, audioe = run()
    finally:
        del dit.__dict__["_sharded_graph_forward"]
    assert dit.shard_graph_stats() == stats                          # the eager run launched no graph
    dit.shard_tokens(None)
    err, aerr = rel_l2(latg, lat1), rel_l2(audiog, audio1)
    report(case="generate_dpmpp_3m_sde", layout="2x2", stats=stats, rel_l2_latents=err, rel_l2_audio=aerr,
           bit_identical=bool(torch.equal(latg, lat1)))
    assert stats[0] >= 1 and stats[1] >= steps - 1, stats           # the sampler's calls were graph launches
    assert torch.equal(latg, late) and torch.equal(audiog, audioe)
    assert err < 4e-3, err
    assert aerr < 4e-3, aerr


def _sa2_length_vs_oracle(rows):
    from oracle import dit_oracle as do
    cfg = dict(SAO_DIT, depth=2)
    sd = do.make_dit_weights(cfg, seed=24)
    g = torch.Generator().manual_seed(25)
    x, t = torch.randn(1, 64, 6144, generator=g), torch.tensor([0.3])
    c, ge = torch.randn(1, 130, 768, generator=g), torch.randn(1, 1536, generator=g)
    yc = do.dit_inner_forward(sd, cfg, x, t, c, ge)
    yu = do.dit_inner_forward(sd, cfg, x, t, torch.zeros_like(c), ge)
    ref = yu + (yc - yu) * 7.0
    m = build_native_dit(cfg, sd).shard_tokens(rows)
    kw = dict(x=x.cuda(), t=t.cuda(), cross_attn_cond=c.cuda(), global_embed=ge.cuda(), cfg_scale=7.0)
    ye = _call(m, kw, False)
    yg = _call(m, kw, True)
    err = rel_l2(ye.cpu(), ref)
    report(case="sa2_length_2_blocks_cfg7", rows=rows, rel_l2=err, stats=m.shard_graph_stats())
    assert torch.equal(yg, ye)
    assert err < 2e-3 * 7.0 / 1.5, err


def _real_rows(world):
    n = torch.cuda.device_count()
    if n < 2 * world:
        pytest.skip(f"{n} CUDA device(s) visible: a CFG split over distinct GPUs with {world} per row needs {2 * world}")
    return [[f"cuda:{i}" for i in range(world)], [f"cuda:{world + i}" for i in range(world)]]


def test_sa2_length_cfg_split_over_2_devices_vs_oracle():
    _sa2_length_vs_oracle(_real_rows(1))


def test_sa2_length_cfg_split_over_4_devices_vs_oracle():
    _sa2_length_vs_oracle(_real_rows(2))
