"""What the Runner hands the optimizer tail, without a GPU (the CPU stand-in of tests/cpu_backend.py): the (lr, step) that reaches
ops.adam_ema (host-fed, data-parallel and per-operator steps) and ops.train_sweep (the single-GPU step) across ExpDecay's decay_start and
its 10 000-step intervals, against a restatement of the reference's step order (runner/runner.py:75-76): ExpDecay.step decides the
learning-rate factor from its count before incrementing it (optims/expdecay.py), jt.nn.Adam.step increments n_step and uses it, then
EMA.ema_step increments its own count, which equals n_step (optims/ema.py).  A checkpoint saved and loaded at a boundary keeps the
sequence, in both formats."""
import pytest
import torch

from test_runner_cpu import make_runner

BOUNDARIES = [20000, 30000, 40000]                 # ExpDecay counts at which lego_cfg's factor is multiplied by 0.33


class ReferenceSchedule:
    """optims/expdecay.py + jt.nn.Adam + optims/ema.py under lego_cfg, one training step at a time"""

    def __init__(self, base_lr=0.1, decay_start=20000, decay_interval=10000, decay_base=0.33, decay_end=10000000):
        self.base_lr, self.decay_start, self.decay_interval, self.decay_base, self.decay_end = base_lr, decay_start, decay_interval, decay_base, decay_end
        self.steps, self.factor, self.n_step, self.ema_steps = 0, 1, 0, 0

    def step(self):
        if self.steps >= self.decay_start and (self.steps - self.decay_start) % self.decay_interval == 0 and self.steps <= self.decay_end:
            self.factor *= self.decay_base
        lr = self.base_lr * self.factor
        self.n_step += 1                           # jt.nn.Adam.step
        self.steps += 1
        self.ema_steps += 1                        # EMA.ema_step
        assert self.ema_steps == self.n_step
        return lr, self.n_step


def _record(monkeypatch, r, sweep):
    """Route the Runner's optimizer calls into a list of (op, lr, step); sweep=True makes it take the single-GPU train_sweep path."""
    from jnerf_b200 import ops
    calls = []
    monkeypatch.setattr(ops, "adam_ema", lambda *a, **k: calls.append(("adam_ema", a[5], a[6])))
    monkeypatch.setattr(ops, "train_sweep", lambda *a, **k: calls.append(("train_sweep", a[9], a[10])))
    if sweep:
        r._fx, r._w_part, r._bwd_rows = torch.zeros(2, dtype=torch.int64), torch.zeros(1), 1
    return calls


def _set_counters(r, ref):
    r.optimizer.steps, r.optimizer.m_learning_rate_factor = ref.steps, ref.factor
    r.optimizer._nested_optimizer.n_step = ref.n_step
    r.ema_optimizer.steps = ref.ema_steps


def _tails(r, calls, k, sweep):
    """k optimizer tails -> their (lr, step); one train_sweep or three adam_ema calls with the same (lr, step) each"""
    out = []
    for _ in range(k):
        n0 = len(calls)
        r._optimizer_tail()
        got = calls[n0:]
        assert [c[0] for c in got] == (["train_sweep"] if sweep else ["adam_ema"] * 3)
        assert len({c[1:] for c in got}) == 1
        out.append(got[0][1:])
        assert r.ema_optimizer.steps == r.optimizer._nested_optimizer.n_step
    return out


@pytest.mark.parametrize("sweep", [True, False], ids=["train_sweep", "adam_ema"])
def test_lr_and_step_across_the_expdecay_boundaries(monkeypatch, sweep):
    r, _ = make_runner(monkeypatch)
    calls = _record(monkeypatch, r, sweep)
    # from step 1, and from just below each boundary with the counters set as a run that got there would have them
    for start in [0] + [b - 2 for b in BOUNDARIES]:
        ref = ReferenceSchedule()
        for _ in range(start):
            ref.step()
        _set_counters(r, ref)
        expect = [ref.step() for _ in range(5)]
        got = _tails(r, calls, 5, sweep)
        assert got == expect, (start, got, expect)
    # lr changes exactly at Adam steps 20 001, 30 001 and 40 001
    ref = ReferenceSchedule()
    seq = [ref.step() for _ in range(40002)]
    changes = [seq[i][1] for i in range(1, len(seq)) if seq[i][0] != seq[i - 1][0]]
    assert changes == [b + 1 for b in BOUNDARIES]
    # and a run from step 1, with no counters set, hands over the same 40 002 pairs
    ref0 = ReferenceSchedule()
    _set_counters(r, ref0)
    del calls[:]
    assert _tails(r, calls, 40002, sweep) == seq


@pytest.mark.parametrize("fmt", ["ckpt.pt", "params.pkl"])
def test_checkpoint_at_a_boundary_keeps_the_schedule(monkeypatch, tmp_path, fmt):
    r, _ = make_runner(monkeypatch, seed=5)
    calls = _record(monkeypatch, r, False)
    ref = ReferenceSchedule()
    for _ in range(29999):
        ref.step()
    _set_counters(r, ref)
    got = _tails(r, calls, 1, False)                             # ExpDecay's count is 30 000: the next step decays the lr
    expect = [ref.step()] + [ref.step() for _ in range(3)]
    p = str(tmp_path / fmt)
    r.cfg.m_training_step = 30001
    r.save_ckpt(p)
    r2, _ = make_runner(monkeypatch, seed=6)
    calls2 = _record(monkeypatch, r2, False)
    r2.load_ckpt(p)
    assert r2.optimizer.steps == 30000 and r2.optimizer._nested_optimizer.n_step == 30000 and r2.ema_optimizer.steps == 30000
    got += _tails(r2, calls2, 3, False)
    assert got == expect, (got, expect)
    assert got[1][1] == 30001 and got[1][0] < got[0][0] and got[2][0] == got[1][0]        # the decay lands on Adam step 30 001
