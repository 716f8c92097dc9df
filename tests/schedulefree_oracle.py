"""A torch restatement of the schedulefree package's ``SGDScheduleFree`` (Defazio et al. 2024, "The Road Less Scheduled"),
foreach branch: the oracle of tests/test_schedulefree.py.  It is written out from the published algorithm op by op, with
the package's group keys, its state ``z`` and its train() / eval() switches; like ``FusedScheduleFreeSGD`` it starts in
eval mode."""
import torch


def schedule(group):
    """The step's (lr, ckp1, alpha_y) in Python floats, committing k + 1 and the running values to ``group``."""
    k = group["k"]
    warmup_steps = group["warmup_steps"]
    if k < warmup_steps:
        sched = (k + 1) / warmup_steps
    else:
        sched = 1.0
    lr = group["lr"] * sched
    lr_max = group["lr_max"] = max(lr, group["lr_max"])
    weight = ((k + 1) ** group["r"]) * (lr_max ** group["weight_lr_power"])
    weight_sum = group["weight_sum"] = group["weight_sum"] + weight
    try:
        ckp1 = weight / weight_sum
    except ZeroDivisionError:
        ckp1 = 0
    group["scheduled_lr"] = lr
    group["k"] = k + 1
    return lr, ckp1, lr * (group["momentum"] * (1 - ckp1) - 1)


class SGDScheduleFreeReference(torch.optim.Optimizer):
    def __init__(self, params, lr=1.0, momentum=0.9, weight_decay=0, warmup_steps=0, r=0.0, weight_lr_power=2.0):
        defaults = dict(lr=lr, momentum=momentum, r=r, k=0, warmup_steps=warmup_steps, train_mode=False,
                        weight_sum=0.0, lr_max=-1.0, scheduled_lr=0.0, weight_lr_power=weight_lr_power,
                        weight_decay=weight_decay, foreach=True)
        super().__init__(params, defaults)

    @torch.no_grad()
    def eval(self):
        for group in self.param_groups:
            if group["train_mode"]:
                for p in group["params"]:
                    if "z" in self.state[p]:
                        p.lerp_(end=self.state[p]["z"], weight=1 - 1 / group["momentum"])
                group["train_mode"] = False

    @torch.no_grad()
    def train(self):
        for group in self.param_groups:
            if not group["train_mode"]:
                for p in group["params"]:
                    if "z" in self.state[p]:
                        p.lerp_(end=self.state[p]["z"], weight=1 - group["momentum"])
                group["train_mode"] = True

    @torch.no_grad()
    def step(self, closure=None):
        if not self.param_groups[0]["train_mode"]:
            raise RuntimeError("not in train mode")
        for group in self.param_groups:
            momentum, weight_decay = group["momentum"], group["weight_decay"]
            lr, ckp1, alpha_y = schedule(group)
            active = [p for p in group["params"] if p.grad is not None]
            for p in active:
                if "z" not in self.state[p]:
                    self.state[p]["z"] = torch.clone(p, memory_format=torch.preserve_format)
            if not active:
                continue
            y = [p for p in active]
            grad = [p.grad for p in active]
            z = [self.state[p]["z"] for p in active]
            if weight_decay != 0:
                torch._foreach_add_(grad, y, alpha=weight_decay)
            torch._foreach_lerp_(y, z, weight=ckp1)
            torch._foreach_add_(y, grad, alpha=lr * (momentum * (1 - ckp1) - 1))
            torch._foreach_sub_(z, grad, alpha=lr)
        return None
