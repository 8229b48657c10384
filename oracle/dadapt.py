"""TEST INFRASTRUCTURE -- restatement of ``dadaptation.DAdaptAdam`` (dadaptation==3.2).

The reference pins ``dadaptation==3.2`` (pyproject.toml:12) and
calls ``dadaptation.DAdaptAdam(self.parameters(), decouple=True)``
(vamb/encode.py:578).  The upstream source is neither in
the reference tree nor a dependency of this project: this file restates
the published algorithm (Defazio & Mishchenko, "Learning-Rate-Free Learning by
D-Adaptation", ICML 2023, Algorithm "Adam with D-Adaptation"; upstream file
``dadaptation/dadapt_adam.py`` of facebookresearch/dadaptation v3.x).

PARITY UNPINNED: no golden vector of the upstream optimiser exists offline.  The
reference tests that exercise this boundary only check that the loss falls
(test/test_encode.py:152-168).  Every parity report that involves
the optimiser therefore says "vs the restated DAdaptAdam".

Hyper-parameters as the reference uses them: lr=1.0, betas=(0.9, 0.999),
eps=1e-8, weight_decay=0, d0=1e-6, growth_rate=inf, use_bias_correction=False,
decouple=True (inert because weight_decay == 0).
"""
from __future__ import annotations

import torch


class DAdaptAdam(torch.optim.Optimizer):
    def __init__(
        self,
        params,
        lr: float = 1.0,
        betas=(0.9, 0.999),
        eps: float = 1e-8,
        weight_decay: float = 0.0,
        log_every: int = 0,
        decouple: bool = False,
        use_bias_correction: bool = False,
        d0: float = 1e-6,
        growth_rate: float = float("inf"),
        fsdp_in_use: bool = False,
    ):
        if not 0.0 < d0:
            raise ValueError(f"Invalid d0 value: {d0}")
        if not 0.0 < lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 < eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 0: {betas[0]}")
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 1: {betas[1]}")
        defaults = dict(
            lr=lr,
            betas=betas,
            eps=eps,
            weight_decay=weight_decay,
            d=d0,
            k=0,
            layer_scale=1.0,
            numerator_weighted=0.0,
            log_every=log_every,
            growth_rate=growth_rate,
            use_bias_correction=use_bias_correction,
            decouple=decouple,
            fsdp_in_use=fsdp_in_use,
        )
        super().__init__(params, defaults)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()

        sk_l1 = 0.0
        group = self.param_groups[0]
        use_bias_correction = group["use_bias_correction"]
        numerator_weighted = group["numerator_weighted"]
        beta1, beta2 = group["betas"]
        k = group["k"]
        d = group["d"]
        lr = max(g["lr"] for g in self.param_groups)
        if use_bias_correction:
            bias_correction = ((1 - beta2 ** (k + 1)) ** 0.5) / (1 - beta1 ** (k + 1))
        else:
            bias_correction = 1
        dlr = d * lr * bias_correction
        growth_rate = group["growth_rate"]
        decouple = group["decouple"]
        sqrt_beta2 = beta2 ** 0.5
        numerator_acum = 0.0

        for group in self.param_groups:
            decay = group["weight_decay"]
            eps = group["eps"]
            group_lr = group["lr"]
            r = group["layer_scale"]
            if group_lr not in [lr, 0.0]:
                raise RuntimeError(
                    "Setting different lr values in different parameter groups is only "
                    "supported for values of 0"
                )
            for p in group["params"]:
                if p.grad is None:
                    continue
                grad = p.grad.data
                if decay != 0 and not decouple:
                    grad.add_(p.data, alpha=decay)
                state = self.state[p]
                if "step" not in state:
                    state["step"] = 0
                    state["s"] = torch.zeros_like(p.data).detach()
                    state["exp_avg"] = torch.zeros_like(p.data).detach()
                    state["exp_avg_sq"] = torch.zeros_like(p.data).detach()
                exp_avg, exp_avg_sq = state["exp_avg"], state["exp_avg_sq"]
                s = state["s"]
                if group_lr > 0.0:
                    denom = exp_avg_sq.sqrt().add_(eps)
                    numerator_acum += (
                        r * dlr * torch.dot(grad.flatten(), s.div(denom).flatten()).item()
                    )
                    exp_avg.mul_(beta1).add_(grad, alpha=r * dlr * (1 - beta1))
                    exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
                    s.mul_(sqrt_beta2).add_(grad, alpha=dlr * (1 - sqrt_beta2))
                    sk_l1 += r * s.abs().sum().item()

        numerator_weighted = sqrt_beta2 * numerator_weighted + (1 - sqrt_beta2) * numerator_acum
        d_hat = d
        if sk_l1 == 0:
            return loss
        if lr > 0.0:
            d_hat = numerator_weighted / ((1 - sqrt_beta2) * sk_l1)
            d = max(d, min(d_hat, d * growth_rate))

        for group in self.param_groups:
            group["numerator_weighted"] = numerator_weighted
            group["d"] = d
            decay = group["weight_decay"]
            k = group["k"]
            eps = group["eps"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                state = self.state[p]
                state["step"] += 1
                exp_avg, exp_avg_sq = state["exp_avg"], state["exp_avg_sq"]
                denom = exp_avg_sq.sqrt().add_(eps)
                if decay != 0 and decouple:
                    p.data.add_(p.data, alpha=-decay * dlr)
                p.data.addcdiv_(exp_avg, denom, value=-1)
            group["k"] = k + 1
        return loss
