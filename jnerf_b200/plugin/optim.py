"""Adam / ExpDecay / EMA / LinearLog mirrors (optims/{adam,expdecay,ema}.py, contrib/mipnerf optims/linearlog.py) on top of ONE fused kernel (ngp_adam_ema).

Reference step order (runner/runner.py:75-76): optimizer.step(loss) [ExpDecay -> jt.nn.Adam] then
ema_optimizer.ema_step(), which overwrites the live parameters with the debiased EMA (ema.py:26-37).
Here `Adam.step` runs backward and, when an EMA is attached to the same parameters, defers the parameter update so
that `EMA.ema_step` can apply Adam + EMA + gradient zeroing in a single streaming pass.  Without an EMA the same
kernel runs with decay 0 (pure Adam)."""
import numpy as np
import torch

from .. import ops
from ..utils.registry import OPTIMS


class _ParamState:
    def __init__(self, p):
        self.p = p
        self.m = torch.zeros(p.numel(), dtype=torch.float32, device=p.device)
        self.v = torch.zeros(p.numel(), dtype=torch.float32, device=p.device)
        self.master = p.detach().float().reshape(-1).clone()     # EMA `values` (ema.py:16-19) == fp32 master copy


@OPTIMS.register_module()
class Adam:
    def __init__(self, params, lr=1e-1, eps=1e-15, betas=(0.9, 0.99), weight_decay=0):
        assert weight_decay == 0, "the NGP configs use weight_decay = 0"
        self.params = [p for p in params if p.requires_grad]
        self.lr, self.eps, self.betas = lr, eps, betas
        self.n_step = 0
        self.state = [_ParamState(p) for p in self.params]
        self._ema = None
        self._pending = False

    def zero_grad(self):
        for p in self.params:
            p.grad = None

    def backward(self, loss):
        loss.sum().backward()                    # Jittor differentiates an unreduced loss as its sum (runner.py:74-75)

    def step(self, loss=None):
        if loss is not None:
            self.backward(loss)
        self.n_step += 1
        if self._ema is not None:
            self._pending = True                 # EMA.ema_step() applies the fused update
        else:
            self._apply(ema_decay=0.0)

    def _apply(self, ema_decay, grad_scale=1.0):
        for st in self.state:
            g = st.p.grad
            if g is None:
                continue
            g = g.reshape(-1)
            if st.p.dtype == torch.float32 and g.dtype != torch.float32:
                g = g.float()
            ops.adam_ema(st.p.data.view(-1), g, st.m, st.v, st.master, self.lr, self.n_step, self.betas[0], self.betas[1], self.eps,
                         ema_decay, grad_scale=grad_scale, zero_grad=False)
            st.p.grad = None
        self._pending = False

    def state_dict(self):
        return {"n_step": self.n_step, "lr": self.lr, "m": [s.m for s in self.state], "v": [s.v for s in self.state],
                "master": [s.master for s in self.state]}

    def load_state_dict(self, sd):
        self.n_step, self.lr = sd["n_step"], sd["lr"]
        for s, m, v, ms in zip(self.state, sd["m"], sd["v"], sd["master"]):
            s.m.copy_(m); s.v.copy_(v); s.master.copy_(ms)


@OPTIMS.register_module()
class ExpDecay:
    """optims/expdecay.py:7-31: lr *= decay_base every decay_interval steps from decay_start on."""

    def __init__(self, nested_optimizer, decay_start, decay_interval, decay_base, decay_end=None):
        self.base_lr = nested_optimizer.lr
        self._nested_optimizer = nested_optimizer
        self.decay_start, self.decay_interval, self.decay_base = decay_start, decay_interval, decay_base
        self.decay_end = 10000000 if decay_end is None else decay_end
        self.steps = 0
        self.m_learning_rate_factor = 1

    def advance_lr(self):
        if self.steps >= self.decay_start and (self.steps - self.decay_start) % self.decay_interval == 0 and self.steps <= self.decay_end:
            self.m_learning_rate_factor *= self.decay_base
        self._nested_optimizer.lr = self.base_lr * self.m_learning_rate_factor
        self.steps += 1
        return self._nested_optimizer.lr

    def step(self, loss=None):
        self.advance_lr()
        self._nested_optimizer.step(loss)

    def zero_grad(self):
        return self._nested_optimizer.zero_grad()

    def state_dict(self):
        return {"steps": self.steps, "m_learning_rate_factor": self.m_learning_rate_factor}

    def load_state_dict(self, sd):
        self.steps, self.m_learning_rate_factor = sd["steps"], sd["m_learning_rate_factor"]


@OPTIMS.register_module()
class EMA:
    """optims/ema.py:7-38."""

    def __init__(self, params, decay, adam=None):
        self.decay = decay
        self.steps = 0
        self.params = [p for p in params if p.requires_grad]
        self._adam = adam
        if adam is not None:
            adam._ema = self

    def attach(self, adam):
        inner = getattr(adam, "_nested_optimizer", adam)
        assert [id(p) for p in inner.params] == [id(p) for p in self.params], "EMA and Adam must cover the same parameters"
        self._adam = inner
        inner._ema = self

    def ema_step(self, loss=None):
        assert loss is None
        self.steps += 1
        assert self._adam is not None and self._adam._pending, "EMA.ema_step must follow optimizer.step (runner.py:75-76)"
        assert self.steps == self._adam.n_step
        self._adam._apply(ema_decay=self.decay)

    def state_dict(self):
        return {"steps": self.steps, "decay": self.decay}

    def load_state_dict(self, sd):
        self.steps = sd["steps"]


@OPTIMS.register_module()
class LinearLog:
    """contrib/mipnerf optims/linearlog.py:8-38: lr = delay * exp(log(start_lr) (1 - t) + log(end_lr) t), t = clip(step / max_steps, 0, 1),
    delay = lr_delay_mult + (1 - lr_delay_mult) sin(pi/2 clip(step / lr_delay_steps, 0, 1)) (1 without a delay), in fp32 as Jittor
    evaluates it.  start_lr is the nested optimizer's lr, as in the reference (its start_lr argument is not read)."""

    def __init__(self, nested_optimizer, start_lr=5e-4, end_lr=5e-6, max_steps=40000, lr_delay_steps=0, lr_delay_mult=1):
        self._nested_optimizer = nested_optimizer
        self.start_lr, self.end_lr, self.max_steps = nested_optimizer.lr, end_lr, max_steps
        self.lr_delay_steps, self.lr_delay_mult = lr_delay_steps, lr_delay_mult
        self.steps = 0

    def lr_at(self, step):
        f = np.float32
        if self.lr_delay_steps > 0:
            x = f(np.clip(f(step / self.lr_delay_steps), 0, 1))
            delay = f(self.lr_delay_mult) + f(1 - self.lr_delay_mult) * np.sin(f(0.5) * f(np.pi) * x)
        else:
            delay = f(1.0)
        t = f(np.clip(f(step / self.max_steps), 0, 1))
        return float(f(delay * np.exp(np.log(f(self.start_lr)) * (f(1) - t) + np.log(f(self.end_lr)) * t)))

    def advance_lr(self):
        self._nested_optimizer.lr = self.lr_at(self.steps)
        self.steps += 1
        return self._nested_optimizer.lr

    def step(self, loss=None):
        self.advance_lr()
        self._nested_optimizer.step(loss)

    def zero_grad(self):
        return self._nested_optimizer.zero_grad()

    def state_dict(self):
        return {"steps": self.steps}

    def load_state_dict(self, sd):
        self.steps = sd["steps"]


@OPTIMS.register_module()
class PlenOptimRMSprop:
    """contrib/plenoxel optims/svox2_optim.py:59-81: Jittor's nn.RMSprop with one group for the density and one for the SH, dense over
    every entry: v = alpha v + (1 - alpha) g^2, p -= lr g / (sqrt(v) + eps) (Jittor's documented RMSprop; DESIGN.md section 12).  It owns
    the gradients, as Jittor's optimizer does: int64 fixed-point sums (ops.SVOX_FX_UNIT a unit) that the training kernels add into and
    step() reads and clears, and the device flag those kernels set when a term or sum leaves the fixed-point range."""

    def __init__(self, p_density, p_sh, lr_sigma, lr_sh, alpha_sigma, alpha_sh, eps=1e-8):
        self.p_density, self.p_sh = p_density, p_sh
        self.lr_sigma, self.lr_sh, self.alpha_sigma, self.alpha_sh, self.eps = lr_sigma, lr_sh, alpha_sigma, alpha_sh, eps
        dev = p_density.device
        self.rms_density, self.rms_sh = torch.zeros_like(p_density), torch.zeros_like(p_sh)
        self.grad_density = torch.zeros(p_density.shape, dtype=torch.int64, device=dev)
        self.grad_sh = torch.zeros(p_sh.shape, dtype=torch.int64, device=dev)
        self.flag = torch.zeros(1, dtype=torch.int32, device=dev)

    def update_lr(self, lr_sigma, lr_sh, alpha_sigma, alpha_sh):
        self.lr_sigma, self.lr_sh, self.alpha_sigma, self.alpha_sh = lr_sigma, lr_sh, alpha_sigma, alpha_sh

    def zero_grad(self):
        self.grad_density.zero_()
        self.grad_sh.zero_()

    def step(self):
        ops.svox_rmsprop(self.p_density, self.p_sh, self.grad_density, self.grad_sh, self.rms_density, self.rms_sh, self.lr_sigma, self.lr_sh,
                         self.alpha_sigma, self.alpha_sh, self.eps)

    def check_overflow(self):
        """Raises if a gradient left the fixed-point range since the optimizer was built (reads the device flag: a synchronisation)."""
        if int(self.flag.item()):
            raise FloatingPointError("PlenOptimRMSprop: a gradient term or sum left the 64-bit fixed-point range (or was not finite)")
