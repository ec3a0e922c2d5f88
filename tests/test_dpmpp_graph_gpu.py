"""The fused CFG + DPM-Solver++ step (dwm_b200_cfg_dpmpp_step) and the CUDA-graph replay of the
CTSD-2.1 step with DPM-Solver++: the kernel is bit-equal to the chain of lincomb2 launches it
replaces, the scheduler's 10-step trajectory to that chain as the scheduler used to run it, and
the graphed UNet step and pipelines stay within the eager run-to-run spread."""
import pytest
import torch

from test_pipeline_gpu import COMMON, _batch
from test_unet import UCFG, _inputs, _oracle

pytestmark = pytest.mark.gpu
SD21 = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012,
            beta_schedule="scaled_linear", steps_offset=1)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _bit_equal(a, b):
    return torch.equal(_bits(a), _bits(b))


def _chain(pred, lat, hist, row, cfg, g):
    """The launches the fused kernel replaces: the pipeline's CFG lincomb2, then the three
    lincomb2 launches of the former DPMSolverMultistepScheduler.step.  Returns (latents, x0)."""
    from opendwm_b200 import ops
    n = lat.numel()
    m = pred
    if cfg == 2:
        m = ops.lincomb2(pred[:n], pred[n:], torch.tensor([1.0 - g], device="cuda"),
                         torch.tensor([g], device="cuda"), torch.empty_like(lat))
    x0 = ops.lincomb2(lat, m, row[0:1], row[1:2], torch.empty_like(lat))
    p = ops.lincomb2(lat, x0, row[2:3], row[3:4], torch.empty_like(lat))
    if row[5].item() == 2:
        p = ops.lincomb2(p, hist, torch.ones(1, device="cuda"), row[4:5], torch.empty_like(lat))
    return p, x0


def _rows():
    """Coefficient rows of the CTSD-2.1 DPM-Solver++ table (both variants, early and late
    steps) and one arbitrary row per order."""
    from dwm.schedulers.dpm_solver import DPMSolverMultistepScheduler
    s = DPMSolverMultistepScheduler(prediction_type="v_prediction", **SD21)
    s.set_timesteps(50, "cuda")
    rows = [s._coef[i, v] for i, v in ((0, 0), (1, 1), (25, 1), (48, 1), (49, 0))]
    g = torch.Generator().manual_seed(3)
    for order in (1.0, 2.0):
        r = torch.randn(6, generator=g)
        r[5] = order
        rows.append(r.cuda())
    return rows


@pytest.mark.parametrize("n", [1, 3, 257, 1001, 2 * 6 * 4 * 32 * 56 + 3])
@pytest.mark.parametrize("cfg", [1, 2])
@pytest.mark.parametrize("g", [1.0, 3.0])
def test_kernel_bit_equal_to_lincomb2_chain(n, cfg, g):
    from opendwm_b200 import ops
    gen = torch.Generator().manual_seed(n + cfg)
    pred = torch.randn(cfg * n, generator=gen)
    lat = torch.randn(n, generator=gen)
    hist = torch.randn(n, generator=gen)
    for t in (pred, lat, hist):           # signed zeros: every fourth element (some of each)
        t[::4] = -0.0
        t[1::8] = 0.0
    pred, lat, hist = pred.cuda(), lat.cuda(), hist.cuda()
    for row in _rows():
        # a first-order step must not read the history: poison it
        h = hist.clone() if row[5].item() == 2 else torch.full_like(hist, float("nan"))
        want, want_x0 = _chain(pred, lat, h, row, cfg, g)
        got, got_h = lat.clone(), h.clone()
        ops.cfg_dpmpp_step(pred, got, got_h, row, cfg=cfg, guidance_scale=g)
        assert _bit_equal(got, want), row.tolist()
        assert _bit_equal(got_h, want_x0), row.tolist()
        assert torch.isfinite(got).all()


def test_kernel_rejects_bad_tensors():
    from opendwm_b200 import ops
    lat, h = torch.zeros(10, device="cuda"), torch.zeros(10, device="cuda")
    row = torch.zeros(6, device="cuda")
    with pytest.raises(ValueError, match="cfg"):
        ops.cfg_dpmpp_step(torch.zeros(10, device="cuda"), lat, h, row, cfg=2)
    with pytest.raises(ValueError, match="6 values"):
        ops.cfg_dpmpp_step(torch.zeros(10, device="cuda"), lat, h, row[:5], cfg=1)
    with pytest.raises(RuntimeError, match="must not overlap"):
        ops.cfg_dpmpp_step(torch.zeros(10, device="cuda"), lat, lat, row, cfg=1)


def _old_scheduler_chain(coef, order, x, preds):
    """DPMSolverMultistepScheduler.step as three lincomb2 launches and a Python history list,
    over a whole schedule of len(preds) < 15 steps (lower_order_final: the last step is first
    order).  Returns the latents after every step."""
    from opendwm_b200 import ops
    n = len(preds)
    hist, lower, out = [None] * order, 0, []
    one = torch.ones(1, device="cuda")
    for i, m in enumerate(preds):
        first = order == 1 or lower < 1 or i == n - 1
        co = coef[i, 0 if first else 1]
        x0 = ops.lincomb2(x, m, co[0:1], co[1:2], torch.empty_like(x))
        hist = hist[1:] + [x0]
        prev = ops.lincomb2(x, x0, co[2:3], co[3:4], torch.empty_like(x))
        if not first:
            prev = ops.lincomb2(prev, hist[-2], one, co[4:5], torch.empty_like(x))
        lower = min(lower + 1, order)
        x = prev
        out.append(x)
    return out


@pytest.mark.parametrize("ptype", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("order", [1, 2])
def test_scheduler_step_bit_equal_to_old_chain(ptype, order):
    from dwm.schedulers.dpm_solver import DPMSolverMultistepScheduler
    s = DPMSolverMultistepScheduler(prediction_type=ptype, solver_order=order, **SD21)
    s.set_timesteps(10, "cuda")
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(1, 2, 3, 4, 8, 6, generator=gen).cuda()
    preds = [(torch.randn(x.shape, generator=gen) * 0.3).cuda() for _ in range(10)]
    want = _old_scheduler_chain(s._coef, order, x.flatten(), [p.flatten() for p in preds])
    x_in, xs = x.clone(), x
    for i in range(10):
        xs = s.step(preds[i], s.timesteps[i], xs).prev_sample
        assert xs.shape == x.shape and xs.dtype == torch.float32
        assert _bit_equal(xs.flatten(), want[i]), i
    assert s.lower_order_nums == order and s._step_index == 10
    assert torch.equal(x, x_in)          # step leaves its sample alone
    # a new schedule starts at first order again
    s.set_timesteps(10, "cuda")
    assert s.lower_order_nums == 0 and s._step_index == 0
    assert _bit_equal(s.step(preds[0], None, x).prev_sample.flatten(), want[0])


def _unet_pipe(inference, fp8=False):
    from dwm.models.crossview_temporal_unet import UNetCrossviewTemporalConditionModel as U
    from dwm.pipelines.ctsd import CrossviewTemporalSD
    o = _oracle(UCFG)
    m = U(**UCFG, compute_dtype=torch.float16,
          gemm_dtype=torch.float8_e4m3fn if fp8 else None)
    m.load_state_dict(o.state_dict())
    inf = dict(inference, scheduler="diffusers.DPMSolverMultistepScheduler")
    pipe = CrossviewTemporalSD(None, {"generator_seed": 0}, "cuda",
                               dict(COMMON, frame_prediction_style="ctsd"), {}, inf, None, m,
                               model_dtype=torch.float32)
    assert type(pipe.test_scheduler).__name__ == "DPMSolverMultistepScheduler"
    return pipe


def _count_replays(monkeypatch):
    count = [0]
    replay = torch.cuda.CUDAGraph.replay

    def counted(self):
        count[0] += 1
        return replay(self)
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", counted)
    return count


def _within_spread(a, a2, b):
    """b (graphed) differs from a (eager) by no more than two eager runs differ (GroupNorm
    statistics are fp64 atomics, so the UNet step is reproducible only to rounding)."""
    assert torch.isfinite(a).all() and torch.isfinite(b).all()
    noise = (a - a2).abs().max().item()
    diff = (a - b).abs().max().item()
    assert diff <= max(4 * noise, 2e-2 * a.abs().max().item()), (diff, noise)


def _counters(s):
    return s._step_index, s.lower_order_nums


def test_unet_step_graphed_with_dpm_solver(monkeypatch):
    """denoise_step_graphed captures the DPM-Solver++ step once for the whole schedule, stays
    within the eager spread, keeps the scheduler's counters in step with an eager run and, after
    set_timesteps, restarts at first order without a new capture."""
    pipe = _unet_pipe({"guidance_scale": 3.0, "inference_steps": 6})
    kind = type(pipe.test_scheduler)
    kw = dict(SD21, clip_sample=False, set_alpha_to_one=False, prediction_type="v_prediction")
    sa, sa2, sb = pipe.test_scheduler, kind(**kw), kind(**kw)
    for s in (sa, sa2, sb):
        s.set_timesteps(6, "cuda")
    x, _, c = _inputs(2, 2, 2)
    c = {k: (v.cuda() if v is not None else None) for k, v in c.items()}
    a, a2, b = (x[:1].clone().cuda() for _ in range(3))
    replays = _count_replays(monkeypatch)

    def step(s, lat, graphed, t):
        pipe.test_scheduler = s
        ts = torch.full((1, 2, 2), t, dtype=torch.int32, device="cuda")
        (pipe.denoise_step_graphed if graphed else pipe.denoise_step)(lat, c, None, ts, None)

    for i, t in enumerate(sa.timesteps.tolist()):
        step(sa, a, False, t)
        step(sa2, a2, False, t)
        step(sb, b, True, t)
        assert _counters(sb) == _counters(sa)
        # the replay ran the step's row: first order on the first and (n < 15) last step
        assert _bit_equal(sb._row, sa._coef[i, 0 if i in (0, 5) else 1]), i
    assert len(pipe._graphs) == 1 and replays[0] == 6
    assert not torch.equal(a, x[:1].cuda())
    _within_spread(a, a2, b)
    # second window on the same buffers: fresh history, first order, the same graph
    for s in (sa, sa2, sb):
        s.set_timesteps(6, "cuda")
        assert _counters(s) == (0, 0)
    t0 = sa.timesteps[0].item()
    step(sa, a, False, t0)
    step(sa2, a2, False, t0)
    step(sb, b, True, t0)
    assert sb._row[5].item() == 1.0 and _counters(sb) == _counters(sa) == (1, 1)
    assert len(pipe._graphs) == 1 and replays[0] == 7
    _within_spread(a, a2, b)


def _run(pipe, method, graphed, *args):
    pipe.inference_config["cuda_graph"] = graphed
    pipe.generator.manual_seed(0)
    pipe.__dict__.pop("_graphs", None)
    out = getattr(pipe, method)(*args)
    return out["latents"] if method == "inference_pipeline" else out["images"]


@pytest.mark.parametrize("fp8", [False, True], ids=["16bit", "e4m3"])
@pytest.mark.parametrize("method", ["inference_pipeline", "autoregressive_inference_pipeline"])
def test_pipelines_replay_dpm_solver_graphs(monkeypatch, method, fp8):
    """cuda_graph: true replays one graph per step (one capture per window) for the CTSD-2.1
    examples' scheduler, and matches cuda_graph: false within the eager spread."""
    steps, T, V = 5, 2, 3
    pipe = _unet_pipe({"guidance_scale": 3.0, "inference_steps": steps,
                       "sequence_length_per_iteration": T, "reference_frame_count": 1}, fp8)
    shape = (1, T, V, 4, 16, 24)
    frames = T if method == "inference_pipeline" else T + 1       # two windows
    batch = _batch(frames, V, dict(joint_attention_dim=96, pooled_projection_dim=8),
                   hw=(128, 192))
    a = _run(pipe, method, False, shape, batch, "pt")
    a2 = _run(pipe, method, False, shape, batch, "pt")
    replays = _count_replays(monkeypatch)
    b = _run(pipe, method, True, shape, batch, "pt")
    windows = frames - T + 1
    assert replays[0] == steps * windows
    assert _counters(pipe.test_scheduler) == (steps, 2)
    assert b.shape == a.shape
    _within_spread(a, a2, b)
