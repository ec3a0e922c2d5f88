"""The opt-in FP8 (E4M3) GEMM path on the GPU: the row quantizer and the E4M3 LayerNorm output
against the CPU restatement, the FP8 GEMM epilogues against float64 on the dequantized
operands, and the DiT forward with gemm_dtype=torch.float8_e4m3fn against the fake-quant
oracle, across kernel variants, CUDA graphs and frame sharding."""
import pytest
import torch

import fp8_emulation as fe
from common import TINY, seeded_oracle, synthetic_inputs

pytestmark = pytest.mark.gpu
F8 = torch.float8_e4m3fn


def _mk(shape, dtype=torch.float32, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


def _q(x):
    from opendwm_b200 import ops
    return ops.quantize_rows(x)


def _dq(q, s):
    return q.double() * s.double()[:, None]


def _relerr(y, ref):
    return ((y.double() - ref).abs().max() / ref.abs().max()).item()


# ------------------------------------------------------------------ quantize_rows
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("K", [64, 1536, 6144])
def test_quantize_rows_bit_exact(dtype, K):
    M = 333
    g = torch.Generator().manual_seed(K)
    x = torch.randn(M, K, generator=g) * torch.exp2(torch.randint(-12, 6, (M, 1), generator=g).float())
    x[0] = 0                              # all zero: scale 1, q 0
    x[1] = 0
    x[1, K // 3] = -7.25                  # single non-zero: -448
    x[2, :] = 1e-3
    x[2, 5] = 3.0                         # one large value, the rest deep in the subnormals
    x[3] = torch.linspace(-1, 1, K)       # reaches -448 and +448
    x = x.to(dtype)
    q, s = _q(x.cuda())
    q_ref, s_ref = fe.quantize_rows(x)
    assert torch.equal(s.cpu(), s_ref)
    assert torch.equal(q.cpu().view(torch.uint8), q_ref.view(torch.uint8))
    assert s[0] == 1 and not q[0].float().any()
    assert q[1, K // 3].float() == -448 and q[3].float().min() == -448 and q[3].float().max() == 448


def test_quantize_rows_pitched_and_errors():
    from opendwm_b200 import ops
    x = _mk((100, 96), torch.bfloat16)[:, :64]
    out = torch.full((100, 80), 0.5, device="cuda").to(F8)
    q, s = ops.quantize_rows(x, out[:, :64])
    q_ref, s_ref = fe.quantize_rows(x.cpu())
    assert torch.equal(q.cpu().view(torch.uint8), q_ref.view(torch.uint8))
    assert torch.equal(s.cpu(), s_ref)
    assert (out[:, 64:].float() == 0.5).all()      # the pitch padding is left alone
    with pytest.raises(RuntimeError, match="multiples of 16"):
        ops.quantize_rows(_mk((10, 24), torch.bfloat16))


# ------------------------------------------------------------------ LayerNorm -> E4M3
@pytest.mark.parametrize("staged", [0, 1])
@pytest.mark.parametrize("mode", ["plain", "modulated", "dual", "add_item"])
def test_layernorm_fp8_output(mode, staged):
    from opendwm_b200 import lib, ops
    M, D, rpi = 4200, 1536, 700                    # >= 4096 rows: eligible for the staged kernel
    items = M // rpi
    x = _mk((M, D), seed=1) * 3 + 1
    kw, ref_in = {}, x.double().cpu()
    w = b = None
    if mode in ("plain", "add_item"):
        w, b = 1 + 0.1 * _mk((D,), seed=2), 0.1 * _mk((D,), seed=3)
        kw.update(weight=w, bias=b)
    if mode == "add_item":
        ai = _mk((items, D), seed=4)
        kw.update(add_item=ai, rows_per_item=rpi)
        ref_in = ref_in + ai.double().cpu().repeat_interleave(rpi, 0)
    mods = {}
    if mode in ("modulated", "dual"):
        for i, k in enumerate(("shift", "scale", "shift2", "scale2")):
            mods[k] = 0.5 * _mk((items, D), seed=10 + i)
        kw.update(shift=mods["shift"], scale=mods["scale"], rows_per_item=rpi)
    out = torch.empty(M, D, device="cuda", dtype=F8)
    sc = torch.empty(M, device="cuda")
    if mode == "dual":
        out2 = torch.empty(M, D, device="cuda", dtype=F8)
        sc2 = torch.empty(M, device="cuda")
        kw.update(shift2=mods["shift2"], scale2=mods["scale2"], out2=out2, out2_scale=sc2)
    lib.set_option("ln_staged", staged)
    try:
        ops.layernorm(x, out, eps=1e-6, out_scale=sc, **kw)
    finally:
        lib.set_option("ln_staged", 1)
    t = ref_in
    n = (t - t.mean(1, keepdim=True)) / torch.sqrt(t.var(1, unbiased=False, keepdim=True) + 1e-6)
    if w is not None:
        n = n * w.double().cpu() + b.double().cpu()

    def mod(sh, scl):
        return n * (1 + mods[scl].double().cpu().repeat_interleave(rpi, 0)) + \
            mods[sh].double().cpu().repeat_interleave(rpi, 0)

    checks = [(out, sc, mod("shift", "scale") if mods else n)]
    if mode == "dual":
        checks.append((out2, sc2, mod("shift2", "scale2")))
    for q, s, ref in checks:
        amax = ref.abs().amax(1)
        s64 = s.double().cpu()
        assert ((s64 - amax / 448).abs() <= 1e-6 * amax / 448).all()
        xh = _dq(q, s).cpu()
        bound = 2 ** -4 * ref.abs() + 2 ** -10 * s64[:, None] + 1e-6 * amax[:, None]
        assert ((xh - ref).abs() <= bound).all(), ((xh - ref).abs() - bound).max().item()


# ------------------------------------------------------------------ FP8 linear
@pytest.fixture(params=["1cta", "2cta"])
def gemm_variant(request):
    from opendwm_b200 import lib
    lib.set_option("gemm_2cta", 1 if request.param == "2cta" else 0)
    yield request.param
    lib.set_option("gemm_2cta", 1)


SHAPES = [s for s in [
    (128, 256, 64), (128, 256, 128), (256, 512, 1536), (192, 1536, 256),
    (448 * 3, 4608, 1536), (77, 320, 320), (1000, 64, 1536), (130, 288, 72),
    (4096, 6144, 1536), (700, 512, 192), (513, 288, 64),
] if s[2] % 16 == 0]
TOL16 = {torch.bfloat16: 6e-3, torch.float16: 1e-3}


def acc_tol(K):
    """Bound on the FP8 wgmma accumulation error, max|d| / max|ref| against float64 on the
    dequantized operands.  Hopper's FP8 MMA adds its products into the fp32 accumulator with
    fewer mantissa bits than an fp32 add, so the error grows with K: measured on an H100
    (400 W) up to 1.8e-4 at K = 64, 3.9e-4 at K = 256 and 1.3e-3 to 2.4e-3 at K = 1536.
    The first guess, 1e-3 for every K <= 6144, held only up to K ~ 600."""
    return 2e-4 + 2e-6 * K


def tol16(dtype, K):
    return TOL16[dtype] + acc_tol(K)


def _operands(M, N, K, seed=0):
    a8, sa = _q(_mk((M, K), seed=seed + 1))
    w8, sw = _q(_mk((N, K), scale=0.05, seed=seed + 2))
    b = _mk((N,), seed=seed + 3)
    return a8, sa, w8, sw, b, _dq(a8, sa) @ _dq(w8, sw).t()


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_store_and_f32(M, N, K, out_dtype, gemm_variant):
    from opendwm_b200 import lib, ops
    a8, sa, w8, sw, b, acc = _operands(M, N, K)
    ref = acc + b.double()
    y = ops.linear(a8, w8, b, a_scale=sa, w_scale=sw, out_dtype=out_dtype)
    assert y.dtype == out_dtype
    assert _relerr(y, ref) < tol16(out_dtype, K)
    y32 = ops.linear(a8, w8, b, epilogue=lib.EPI_F32, a_scale=sa, w_scale=sw, out_dtype=out_dtype)
    err = _relerr(y32, ref)
    print("fp8 F32 epilogue rel err", (M, N, K), err)
    assert err < acc_tol(K)


@pytest.mark.parametrize("act", ["gelu_tanh", "gelu_erf", "silu", "relu"])
def test_activation(act, gemm_variant):
    from opendwm_b200 import lib, ops
    code = {"gelu_tanh": lib.ACT_GELU_TANH, "gelu_erf": lib.ACT_GELU_ERF, "silu": lib.ACT_SILU,
            "relu": lib.ACT_RELU}[act]
    fn = {"gelu_tanh": lambda z: torch.nn.functional.gelu(z, approximate="tanh"),
          "gelu_erf": torch.nn.functional.gelu, "silu": torch.nn.functional.silu,
          "relu": torch.relu}[act]
    a8, sa, w8, sw, b, acc = _operands(600, 1024, 512)
    ref = fn(acc + b.double())
    for od in (torch.bfloat16, torch.float16):
        y = ops.linear(a8, w8, b, act=code, a_scale=sa, w_scale=sw, out_dtype=od)
        assert _relerr(y, ref) < tol16(od, 512)


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float16])
def test_geglu(out_dtype, gemm_variant):
    from opendwm_b200 import lib, ops
    M, N, K = 700, 1024, 1536
    a8, sa, w8, sw, b, acc = _operands(M, N, K)
    z = (acc + b.double()).view(M, N // 256, 2, 128)
    ref = (z[:, :, 0] * torch.nn.functional.gelu(z[:, :, 1])).reshape(M, N // 2)
    y = ops.linear(a8, w8, b, epilogue=lib.EPI_GEGLU, a_scale=sa, w_scale=sw, out_dtype=out_dtype)
    assert _relerr(y, ref) < tol16(out_dtype, K)


@pytest.mark.parametrize("regions", [1, 2])
def test_qknorm(regions, gemm_variant):
    from opendwm_b200 import lib, ops
    M, D = 600, 256
    a8, sa, w8, sw, b, acc = _operands(M, 3 * D, 512)
    qw, kw = 1 + 0.1 * _mk((64,), seed=7), 1 + 0.1 * _mk((64,), seed=8)
    z = acc + b.double()
    ref = z.clone()
    for r, nw in list(enumerate((qw, kw)))[:regions]:
        h = z[:, r * D:(r + 1) * D].reshape(M, -1, 64)
        h = h * torch.rsqrt((h * h).mean(-1, keepdim=True) + 1e-6) * nw.double()
        ref[:, r * D:(r + 1) * D] = h.reshape(M, D)
    for od in (torch.bfloat16, torch.float16):
        y = ops.linear(a8, w8, b, epilogue=lib.EPI_QKNORM, q_norm_weight=qw, k_norm_weight=kw,
                       qk_region=D, qk_norm_regions=regions, eps=1e-6, a_scale=sa, w_scale=sw,
                       out_dtype=od)
        assert _relerr(y, ref) < tol16(od, 512)


def test_resid_gate_blend(gemm_variant):
    from opendwm_b200 import lib, ops
    M, N, K, rpi = 1200, 512, 1536, 300
    a8, sa, w8, sw, b, acc = _operands(M, N, K)
    resid = _mk((M, N), seed=5)
    gate = _mk((M // rpi, N), seed=6)
    x = _mk((M, N), seed=9)
    alpha = torch.tensor([0.3, 0.8], device="cuda")
    v = (acc + b.double()) * gate.double().repeat_interleave(rpi, 0) + resid.double()
    y = ops.linear(a8, w8, b, epilogue=lib.EPI_RESID, resid=resid, gate=gate, rows_per_item=rpi,
                   a_scale=sa, w_scale=sw, out_dtype=torch.bfloat16)
    assert _relerr(y, v) < acc_tol(K)
    al = alpha.double().repeat_interleave(M // 2)[:, None]
    ref = al * x.double() + (1 - al) * v
    out = x.clone()
    ops.linear(a8, w8, b, epilogue=lib.EPI_RESID, resid=resid, gate=gate, rows_per_item=rpi,
               out=out, blend_x=out, alpha=alpha, rows_per_batch=M // 2, a_scale=sa, w_scale=sw,
               out_dtype=torch.float16)
    assert _relerr(out, ref) < acc_tol(K)


@pytest.mark.parametrize("epi", ["store", "qknorm", "geglu", "resid", "f32"])
def test_kernel_variants_give_identical_bits(epi):
    """1-CTA vs 2-CTA and 128- vs 256-column tiles; peer_out copies equal the local output."""
    from opendwm_b200 import lib, ops
    M, N, K = 1100, 768, 1536
    a8, sa, w8, sw, b, _ = _operands(M, N, K, seed=3)
    resid = _mk((M, N), seed=4)
    kw = dict(a_scale=sa, w_scale=sw, out_dtype=torch.bfloat16)
    kw.update({"store": dict(act=lib.ACT_GELU_TANH),
               "qknorm": dict(epilogue=lib.EPI_QKNORM, q_norm_weight=1 + _mk((64,)) * 0.1,
                              k_norm_weight=1 + _mk((64,), seed=1) * 0.1, qk_region=256),
               "geglu": dict(epilogue=lib.EPI_GEGLU),
               "resid": dict(epilogue=lib.EPI_RESID, resid=resid),
               "f32": dict(epilogue=lib.EPI_F32)}[epi])
    outs = []
    try:
        for cta in (0, 1):
            for bn in ((256,) if epi == "geglu" else (128, 256)):
                lib.set_option("gemm_2cta", cta)
                lib.set_option("gemm_bn", bn)
                if epi in ("store", "qknorm", "geglu"):
                    cols = N // 2 if epi == "geglu" else N
                    out = torch.full((M, cols), float("nan"), device="cuda").to(torch.bfloat16)
                    peers = [torch.full_like(out, float("nan")) for _ in range(2)]
                    ops.linear(a8, w8, b, out=out, peer_out=[p.data_ptr() for p in peers], **kw)
                    for p in peers:
                        assert torch.equal(p, out)
                else:
                    out = ops.linear(a8, w8, b, **kw)
                outs.append(out)
    finally:
        lib.set_option("gemm_2cta", 1)
        lib.set_option("gemm_bn", 0)
    assert not outs[0].float().isnan().any()
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


def test_errors_are_loud():
    from opendwm_b200 import ops
    a8, sa, w8, sw, b, _ = _operands(128, 256, 64)
    with pytest.raises(ValueError, match="a_scale and w_scale"):
        ops.linear(a8, w8, b, a_scale=sa, out_dtype=torch.bfloat16)
    with pytest.raises(TypeError, match="out_dtype"):
        ops.linear(a8, w8, b, a_scale=sa, w_scale=sw)
    a40, s40 = torch.zeros(128, 40, device="cuda", dtype=F8), torch.ones(128, device="cuda")
    w40, t40 = torch.zeros(256, 40, device="cuda", dtype=F8), torch.ones(256, device="cuda")
    with pytest.raises(RuntimeError, match="multiples of 16"):
        ops.linear(a40, w40, a_scale=s40, w_scale=t40, out_dtype=torch.bfloat16)


# ------------------------------------------------------------------ the DiT in FP8
def _fp8_model(cfg, sd, dtype):
    from dwm.models.crossview_temporal_dit import DiTCrossviewTemporalConditionModel
    m = DiTCrossviewTemporalConditionModel(**cfg, compute_dtype=dtype, gemm_dtype=F8)
    m.load_state_dict(sd)
    return m.cuda()


@pytest.mark.parametrize("which", ["tiny", "real_width"])
def test_model_accuracy_against_fake_quant_oracle(which):
    if which == "tiny":
        cfg, std, inp, dtype = TINY, 0.05, {}, torch.float16
    else:
        cfg, std, inp, dtype = dict(TINY, **fe.REAL_WIDTH), fe.REAL_WIDTH_STD, \
            fe.REAL_WIDTH_INPUTS, torch.bfloat16
    o = seeded_oracle(cfg, std=std)
    sample, timestep, cond = synthetic_inputs(cfg, **inp)
    emu, ref, _ = fe.emulated_error(o, sample, timestep, cond)
    m = _fp8_model(cfg, o.state_dict(), dtype)
    dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in cond.items()}
    y = m(sample.cuda(), timestep.cuda(), **dev)[0][0]
    err = fe.rel_err(y.cpu(), ref)
    print("fp8 model error", which, err, "fake-quant oracle", emu,
          "weight bytes saved", m._pk["fp8_bytes_saved"])
    assert err <= 1.5 * emu and err < 0.1, (err, emu)
    # the packed weights are the emulator's: same quantizer on the same fp32 parameters
    at = o.transformer_blocks[0].attn
    w = torch.cat([at.to_q.weight, at.to_k.weight, at.to_v.weight]).detach()
    q_ref, s_ref = fe.quantize_rows(w)
    q, s = m._pk["blocks"][0]["qkv"].w, m._pk["blocks"][0]["qkv"].scale
    assert torch.equal(q.cpu().view(torch.uint8), q_ref.view(torch.uint8))
    assert torch.equal(s.cpu(), s_ref)
    assert m._pk["fp8_bytes_saved"] > 0


def test_model_deterministic_and_graph_equals_eager():
    from dwm.common import create_instance_from_config
    from dwm.pipelines.ctsd import StreamingCrossviewTemporalSD
    o = seeded_oracle(TINY)
    m = create_instance_from_config(
        {"_class_name": "dwm.models.crossview_temporal_dit.DiTCrossviewTemporalConditionModel",
         **TINY, "compute_dtype": {"_class_name": "get_class", "class_name": "torch.float16"},
         "gemm_dtype": {"_class_name": "get_class", "class_name": "torch.float8_e4m3fn"}})
    m.load_state_dict(o.state_dict())
    m.cuda()
    sample, timestep, cond = synthetic_inputs(TINY, device="cuda")
    y1 = m.forward_tokens(sample, timestep, **cond)[0].clone()
    y2 = m.forward_tokens(sample, timestep, **cond)[0].clone()
    assert torch.equal(y1, y2) and torch.isfinite(y1).all()
    pipe = StreamingCrossviewTemporalSD(
        None, {"generator_seed": 0}, "cuda", {"frame_prediction_style": "diffusion_forcing"}, {},
        {"guidance_scale": 2.0, "inference_steps": 12, "sequence_length_per_iteration": 4},
        None, m, model_dtype=torch.float32)
    pipe.reset_streaming((1, 4, 3, 16, 8, 12), "pt")
    a, b = sample[:1].clone().float(), sample[:1].clone().float()
    for i in (9, 10, 11):
        idx, ts, rng = pipe._df_step_tensors(i, 4, 3, 0, 1, 3)
        pipe.denoise_step(a, cond, idx, ts, rng)
        pipe.denoise_step_graphed(b, cond, idx, ts, rng)
    assert len(pipe._graphs) == 1
    assert torch.equal(a, b) and not torch.equal(a, sample[:1])


SHARD_CASES = [(k, T, w) for T, w in ((4, 2), (5, 4)) for k in ("pointwise", "rowwise", "full")]


@pytest.mark.parametrize("use_peer_scatter", [False, True], ids=["allgather", "peer"])
@pytest.mark.parametrize("kind,T,t_ways", SHARD_CASES)
def test_sharded_fp8_forward_equals_unsharded(kind, T, t_ways, use_peer_scatter, monkeypatch):
    from test_sharded_forward_gpu import _AllGatherStub, _PeerExchange, _state_dict
    from opendwm_b200 import lib, sharding
    from opendwm_b200.sharding import ShardPlan
    cfg = dict(TINY, temporal_attention_type=kind)
    sd = _state_dict(kind)
    n_blocks = len(cfg["temporal_block_layers"])
    sample, timestep, cond = synthetic_inputs(cfg, T=T, device="cuda")
    B = sample.shape[0]
    if use_peer_scatter:
        exchange = _PeerExchange(n_blocks)
        monkeypatch.setattr(sharding, "PeerKV", exchange.cls)
    else:
        exchange = _AllGatherStub(n_blocks)
    ranks = []
    for r in range(t_ways):
        plan = ShardPlan(t_ways, r, T, cfg=False, make_groups=False)
        plan.use_peer_scatter = use_peer_scatter
        if not use_peer_scatter:
            exchange.bind(plan)
        m = _fp8_model(cfg, sd, torch.float16)
        m.shard = plan
        fs = plan.frame_slice()
        ranks.append((m, plan, sample[:, fs].contiguous(), timestep[:, fs].contiguous(),
                      plan.local_conditions(cond, cfg_doubled=False)))
    try:
        lib.set_option("attn_tc", 0)
        ref = _fp8_model(cfg, sd, torch.float16).forward_tokens(sample, timestep, **cond)[0].clone()
        prev, settled = None, False
        for _ in range(n_blocks + 2):
            exchange.begin_round()
            parts = []
            for m, plan, s_loc, t_loc, c_loc in ranks:
                tok, _ = m.forward_tokens(s_loc, t_loc, **c_loc, t_offset=plan.t_offset, T_total=T)
                parts.append(tok.view(B, plan.T_loc, -1, tok.shape[1]).clone())
            stitched = torch.cat(parts, 1).reshape(ref.shape)
            if prev is not None and torch.equal(stitched, prev):
                settled = True
                break
            prev = stitched
        torch.cuda.synchronize()
    finally:
        lib.set_option("attn_tc", -1)
    assert settled
    exchange.check_final_round()
    assert torch.equal(stitched, ref), ((stitched - ref).abs().max() / ref.abs().max()).item()


def test_pipeline_with_gemm_dtype_from_config():
    from dwm.common import create_instance_from_config
    from dwm.models.cogvideox_vae import AutoencoderKLCogVideoX
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    from test_pipeline_gpu import COMMON, _batch
    from test_vae_gpu import CFG as VCFG
    cfg = dict(TINY, projection_class_embeddings_input_dim=11 * 256)
    o = seeded_oracle(cfg)
    m = create_instance_from_config(
        {"_class_name": "dwm.models.crossview_temporal_dit.DiTCrossviewTemporalConditionModel",
         **cfg, "compute_dtype": {"_class_name": "get_class", "class_name": "torch.float16"},
         "gemm_dtype": {"_class_name": "get_class", "class_name": "torch.float8_e4m3fn"}})
    m.load_state_dict(o.state_dict())
    torch.manual_seed(0)
    vae = AutoencoderKLCogVideoX(**VCFG, compute_dtype=torch.float16).cuda()
    common = dict(COMMON, frame_prediction_style="ctsd", memory_efficient_batch=2,
                  vae_instance=vae)
    pipe = CrossviewTemporalSD(None, {"generator_seed": 0}, "cuda", common, {},
                               {"guidance_scale": 3.0, "inference_steps": 3}, None, m,
                               model_dtype=torch.float16)
    r = pipe.inference_pipeline((1, 3, 3, 16, 8, 12), _batch(3, 3, cfg), "pt")
    assert m._pk["fp8"]
    assert torch.isfinite(r["latents"]).all() and torch.isfinite(r["images"]).all()
