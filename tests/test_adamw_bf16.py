"""`adamw_bf16` (SURVEY.md §8f rank 1): CPU — the oracle against the reference's own `_make_step` executed verbatim
(tests/golden/adamw_bf16_golden.pt) and the host-side bookkeeping; GPU — the kernel with the golden's integers, bit for
bit against the reference's eager chain on the GPU (the other adamw_* cases of tests/kernel_checks.py extend it), and
the optimizer end to end (internal generator, fused clamp and EMA, one launch per TrainStep)."""
from pathlib import Path

import pytest
import torch

from oracle import adamw_bf16_oracle as A

G = torch.load(Path(__file__).parent / "golden" / "adamw_bf16_golden.pt")
NAMES = ("p", "shift", "exp_avg", "exp_avg_sq")


def _run_oracle(semantics):
    p = G["p0"].clone()
    s, m, v = (torch.zeros_like(p) for _ in range(3))
    hp = G["hp"]
    out = []
    for k, dec in enumerate(G["decays"]):
        A.adamw_bf16_step(p, G[f"step{k}.grad"], s, m, v, beta1=hp["beta1"], beta2=hp["beta2"], step=float(k + 1), lr=hp["lr"],
                          eps=hp["eps"], decay_this_iteration=dec, rnd=list(G[f"step{k}.rnd"]), scalar_semantics=semantics)
        out.append(tuple(t.clone() for t in (p, s, m, v)))
    return out


def test_oracle_is_bit_exact_against_reference_make_step():
    for k, state in enumerate(_run_oracle("cpu")):
        for t, n in zip(state, NAMES):
            assert torch.equal(t, G[f"step{k}.{n}"]), (k, n)


def test_cuda_scalar_semantics_differ_only_where_torch_itself_does():
    """fp32 vs bf16-cast eps / alpha and the addcdiv / addcmul association: exp_avg identical, exp_avg_sq only where
    value * (g * g) and (value * g) * g round differently, p / shift within one bf16 ulp."""
    assoc = []
    for k in range(len(G["decays"])):
        g = G[f"step{k}.grad"].double()
        value = float(torch.tensor(1 - G["hp"]["beta2"], dtype=torch.float32))
        assoc.append((value * g * g).float() != (torch.tensor(value) * g.float()).double().mul(g).float())
    for k, state in enumerate(_run_oracle("cuda")):
        assert torch.equal(state[2], G[f"step{k}.exp_avg"])
        diff = state[3] != G[f"step{k}.exp_avg_sq"]
        assert not (diff & ~torch.stack(assoc[:k + 1]).any(0)).any(), k
        assert float((state[3].float() - G[f"step{k}.exp_avg_sq"].float()).abs().max()) <= \
            float(G[f"step{k}.exp_avg_sq"].float().abs().max()) * 2 ** -7
        assert float((state[0] != G[f"step{k}.p"]).float().mean()) < 0.02
        d = (state[0].float() - G[f"step{k}.p"].float()).abs()
        assert float(d.max()) <= float(G[f"step{k}.p"].float().abs().max()) * 2 ** -7


def test_stochastic_rounding_is_unbiased_and_quirk_is_kept():
    x = torch.full((200000,), 1.0 + 2 ** -10)               # 1/8 of a bf16 ulp above 1
    r = torch.randint(0, 1 << 16, x.shape, dtype=torch.int32, generator=torch.Generator().manual_seed(0))
    y = A.copy_stochastic(x, r).float()
    assert set(y.unique().tolist()) == {1.0, 1.0078125} and abs(float(y.mean()) - float(x[0])) < 2e-5
    # quirk Q-opt: first moment = grad + (1 - beta1) * beta1 * exp_avg_old
    p, g = torch.zeros(4).bfloat16(), torch.full((4,), 0.5).bfloat16()
    s, m, v = torch.zeros(4).bfloat16(), torch.full((4,), 2.0).bfloat16(), torch.zeros(4).bfloat16()
    A.adamw_bf16_step(p, g, s, m, v, beta1=0.5, beta2=0.999, step=1.0, lr=1e-3, eps=1e-6, decay_this_iteration=0.0,
                      rnd=[torch.zeros(4, dtype=torch.int32)] * 4)
    assert torch.allclose(m.float(), torch.full((4,), 0.5 + 0.5 * (0.5 * 2.0)))


def test_decay_schedule_and_block_map():
    from simpletuner_b200.training.optim import build_block_map
    acc, fired = 0.004, []
    for _ in range(6):
        dec, acc = A.decay_schedule(acc, weight_decay=1e-2, lr=0.1)
        fired.append(dec)
    assert fired[0] == 0 and fired[1] > 5e-3 and abs(sum(fired) + acc - (0.004 + 6e-3)) < 1e-12
    bt, bo = build_block_map([5, 2048, 2049, 1], 2048)
    assert bt == [0, 1, 2, 2, 3] and bo == [0, 0, 0, 2048, 0]


@pytest.mark.gpu
def test_cuda_kernel_matches_oracle_with_the_same_random_integers():
    """The golden's gradients and random integers through AdamWBF16's `_rnd`, from a random non-zero state, bit for bit
    against the oracle's `_make_step` op sequence run on copies of the same CUDA tensors (the adamw_golden_rnd check)."""
    from tests.kernel_checks import CHECKS
    r = CHECKS["adamw_golden_rnd"]()
    assert r["ok"], r


@pytest.mark.gpu
def test_optimizer_minimises_a_quadratic_with_internal_rng():
    from simpletuner_b200.training.optim import AdamWBF16
    torch.manual_seed(0)
    target = torch.randn(3000, device="cuda")
    w = torch.nn.Parameter(torch.zeros(3000, device="cuda", dtype=torch.bfloat16))
    opt = AdamWBF16([w], lr=2e-2, weight_decay=0.0, seed=123)
    first = None
    for _ in range(300):
        loss = ((w.float() - target) ** 2).mean()
        first = first if first is not None else float(loss)
        w.grad = (2 * (w.float() - target) / w.numel() * 1000).bfloat16()   # scaled: this optimizer has no 1/sqrt(v) bias fix
        opt.step()
    assert float(((w.float() - target) ** 2).mean()) < 0.05 * first


@pytest.mark.gpu
def test_fused_value_clamp_and_ema_match_the_separate_eager_passes():
    """One launch with grad_clamp + EMA == clip_grad_value_ -> step -> EMAModel.step (trainer.py:7188-7195, 7239,
    7351-7357), bit for bit, with the same stochastic-rounding integers."""
    from simpletuner_b200.training.ema import EMAModel
    from simpletuner_b200.training.optim import AdamWBF16
    dev = "cuda"
    g = torch.Generator().manual_seed(5)
    sizes = [4096, 1003, 8, 70001]
    p0 = [torch.randn(n, generator=g).bfloat16() for n in sizes]

    def make():
        ps = [torch.nn.Parameter(t.clone().to(dev)) for t in p0]
        opt = AdamWBF16(ps, lr=3e-3, weight_decay=0.0, seed=2)
        for p_ in ps:
            opt.state[p_].update(step=0.0, exp_avg=torch.zeros_like(p_), exp_avg_sq=torch.zeros_like(p_), shift=torch.zeros_like(p_),
                                 accumulated_decay=0.0)
        return ps, opt, EMAModel(ps, decay=0.97, ema_update_interval=2)

    (pa, oa, ea), (pb, ob, eb) = make(), make()
    clamp = 0.37                               # not a bf16 number: the clamp result itself rounds
    for k in range(1, 5):
        grads = [torch.randn(n, generator=g).bfloat16() for n in sizes]
        grads[1][5] = float("nan") if k == 3 else grads[1][5]
        rnd = torch.randint(0, 1 << 16, (4, sum(sizes)), generator=g, dtype=torch.int32).to(dev)
        for p_, p2, gr in zip(pa, pb, grads):
            p_.grad, p2.grad = gr.clone().to(dev), gr.clone().to(dev)
        oa.step(_rnd=rnd, grad_clamp=clamp, ema=ea, ema_global_step=k)
        torch.nn.utils.clip_grad_value_(pb, clamp)
        ob.step(_rnd=rnd)
        eb.step(pb, global_step=k)
        torch.cuda.synchronize()
        assert ea.optimization_step == eb.optimization_step and ea.cur_decay_value == eb.cur_decay_value
        for i in range(len(sizes)):
            assert torch.equal(pa[i].grad, grads[i].to(dev)) or k == 3            # the stored gradient is not modified
            same = lambda x, y: torch.equal(torch.nan_to_num(x.float(), nan=7.0), torch.nan_to_num(y.float(), nan=7.0))
            assert same(pa[i], pb[i]) and same(oa.state[pa[i]]["exp_avg"], ob.state[pb[i]]["exp_avg"]), (k, i)
            assert same(ea.shadow_params[i], eb.shadow_params[i]), (k, i)
    assert not torch.equal(ea.shadow_params[0], pa[0])                          # the shadows did move and lag the weights


@pytest.mark.gpu
def test_train_step_routes_clamp_and_ema_through_the_optimizer_launch():
    from simpletuner_b200 import ops
    from simpletuner_b200.training.ema import EMAModel
    from simpletuner_b200.training.optim import AdamWBF16
    from simpletuner_b200.training.step import TrainStep
    w = torch.nn.Parameter(torch.ones(4096, device="cuda", dtype=torch.bfloat16))

    class _M:
        model = None
        def prepare_batch(self, b, s): return b
        def model_predict(self, b): return (w.float() * b["x"]).sum()
        def loss_with_logs(self, b, out, apply_conditioning_mask=True): return out, {}

    ema = EMAModel([w], decay=0.5)
    step = TrainStep(_M(), AdamWBF16([w], lr=1e-2, seed=0), max_grad_norm=0.25, ema=ema)
    n0 = ops.launch_count()
    for _ in range(3):
        step({"x": torch.full((4096,), 3.0, device="cuda")})
    torch.cuda.synchronize()
    assert ops.launch_count() - n0 == 3                                         # one library launch per optimizer step
    assert ema.optimization_step == 3 and float((ema.shadow_params[0].float() - 1).abs().max()) > 0
    # |g| = 3 clamped to 0.25: first-moment quirk (grad + 0.1 * 0.9 * m) keeps m bounded by the clamp, not by 3
    assert float(step.optimizer.state[w]["exp_avg"].float().abs().max()) < 0.3
