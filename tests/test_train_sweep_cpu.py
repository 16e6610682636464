"""The Runner's folded optimizer tail (ops.network_bwd_fx + one ops.train_sweep per step) without a GPU: the CPU stand-in of
tests/cpu_backend.py, extended by stand-ins of the two new operators.  Checks the call sequence of the sequential and the pipelined
step, where the next step's front may start with the step in flight, that the folded step trains exactly as the per-tensor sweeps
do, and that under the plain stand-in (no stand-ins for the new operators) the Runner makes the per-tensor calls."""
import pytest
import torch

import cpu_backend
from test_runner_cpu import make_runner


class _FoldOps:
    """Stand-ins of network_bwd_scratch / network_bwd_fx / train_sweep: the scratch holds the fp16-rounded table gradient as
    fp32 and the weight gradients in one slot, and the sweep hands them to the stand-in adam_ema."""

    def __init__(self, fake):
        self.fake = fake

    def network_bwd_scratch(self, levels, device="cpu"):
        return torch.zeros(levels.n_params, dtype=torch.float32), torch.zeros(3072 + 7168, dtype=torch.float32)

    def network_bwd_fx(self, coords, enc, levels, wd, wr, dout, fx, w_part, n_dev=None):
        gg, dwd, dwr = torch.zeros(levels.n_params, dtype=torch.float16), torch.zeros(3072), torch.zeros(7168)
        self.fake.network_bwd(coords, enc, levels, wd, wr, dout, gg, dwd, dwr, n_dev=n_dev)
        self.fake.calls[-1] = "network_bwd_fx"
        fx += gg.float()
        w_part += torch.cat([dwd, dwr])

    def train_sweep(self, table, ts, fx, w_part, bwd_rows, wd, ws, wr, rs, lr, step, beta1=0.9, beta2=0.99, eps=1e-15, ema_decay=0.95):
        n = len(self.fake.calls)
        for p, g, (m, v, ms) in ((table, fx.half(), ts), (wd, w_part[:3072].clone(), ws), (wr, w_part[3072:].clone(), rs)):
            self.fake.adam_ema(p, g, m, v, ms, lr, step, beta1, beta2, eps, ema_decay)
        del self.fake.calls[n:]
        self.fake.calls.append("train_sweep")
        fx.zero_()
        w_part.zero_()


def _install_fold(monkeypatch):
    """cpu_backend.install plus the folded-tail stand-ins; ops._network_bwd names the stand-in network_bwd, so the Runner folds."""
    real_install = cpu_backend.install

    def install(mp):
        fake = real_install(mp)
        import jnerf_b200.ops as real_ops
        fold = _FoldOps(fake)
        for name in ("network_bwd_scratch", "network_bwd_fx", "train_sweep"):
            mp.setattr(real_ops, name, getattr(fold, name), raising=False)
        mp.setattr(real_ops, "_network_bwd", real_ops.network_bwd)
        return fake
    monkeypatch.setattr(cpu_backend, "install", install)


@pytest.fixture
def fold_backend(monkeypatch):
    _install_fold(monkeypatch)


class _MarkEvent:
    """Stands in for the pipeline's "front of the next step may start" event: logs where it is recorded."""

    def __init__(self, calls):
        self.calls = calls

    def record(self, *a, **k):
        self.calls.append("front may start")


SEQ_OPS = ["prepare_batch", "march", "compact", "network_fwd", "composite_loss_bwd", "network_bwd_fx", "train_sweep"]


def test_folded_sequential_step_is_one_backward_and_one_host_argument_sweep(monkeypatch, fold_backend):
    r, fake = make_runner(monkeypatch)
    assert r._fx is not None
    fake.calls.clear()
    r.train_step()
    assert fake.calls == SEQ_OPS
    fake.calls.clear()
    r.train_step()
    assert fake.calls == SEQ_OPS
    assert not r._fx.any() and not r._w_part.any()                 # the sweep leaves the scratch cleared


def test_folded_pipelined_step_starts_the_next_front_with_the_step(monkeypatch, fold_backend):
    r, fake = make_runner(monkeypatch, pipeline=True)
    assert r._fx is not None and r._pipe["at"] == "front"            # the next front may start as soon as the step in flight does
    r.train_step()
    r._pipe["mid"] = _MarkEvent(fake.calls)
    fake.calls.clear()
    r.train_step()
    step = ["front may start", "network_fwd", "composite_loss_bwd", "network_bwd_fx", "train_sweep", "prepare_batch", "march", "compact"]
    assert fake.calls == step, fake.calls                           # this step's back, then the front of the next step behind the mark
    assert fake.calls.count("train_sweep") == 1 and "adam_ema" not in fake.calls and "network_bwd" not in fake.calls


@pytest.mark.parametrize("pipeline", [False, True], ids=["sequential", "pipelined"])
def test_folded_step_trains_as_the_per_tensor_sweeps(monkeypatch, pipeline):
    r, _ = make_runner(monkeypatch, pipeline=pipeline)
    assert r._fx is None
    for _ in range(3):
        r.train_step()
    plain = {k: v.detach().clone() for k, v in r.model.state_dict().items()}
    _install_fold(monkeypatch)
    r2, _ = make_runner(monkeypatch, pipeline=pipeline)
    assert r2._fx is not None
    for _ in range(3):
        r2.train_step()
    for k, v in r2.model.state_dict().items():
        assert torch.equal(v, plain[k]), k


def test_plain_stand_in_keeps_the_per_tensor_calls(monkeypatch):
    r, fake = make_runner(monkeypatch, pipeline=True)
    assert r._fx is None
    r.train_step()
    fake.calls.clear()
    r.train_step()
    assert fake.calls[:6] == ["network_fwd", "composite_loss_bwd", "network_bwd", "adam_ema", "adam_ema", "adam_ema"], fake.calls
