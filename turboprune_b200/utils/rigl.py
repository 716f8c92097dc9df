"""RigL schedule (Evci et al. 2020, "Rigging the Lottery"): which batches of a level update the masks, and how many
weights each update drops and regrows per layer.  Host arithmetic in float64; the selection itself runs on the GPU
(``ops.rigl_select`` / ``ops.rigl_apply``, through ``pruning_utils.rigl_update``).

Config (``pruning_params``, read with defaults so that ``+pruning_params.<key>=...`` works on any config tree):
``training_type: rigl``, ``rigl_update_interval`` (dT, 100), ``rigl_drop_fraction`` (alpha, 0.3),
``rigl_end_fraction`` (0.75).  Within a level of T batches, batch t (t batches already consumed) is an update batch
when t > 0, t % dT == 0 and t < T_end = floor(end_fraction * T); it moves k_l = floor(f(t) * n_active_l) weights of
layer l, with f(t) = alpha / 2 * (1 + cos(pi t / T_end)).
"""
import math

# the initial mask comes from a one-shot method at level 0 (the at_init path); iterative methods have no place here
RIGL_INIT_METHODS = ("er_erk", "er_balanced", "snip", "synflow")


def is_rigl(cfg) -> bool:
    return getattr(cfg.pruning_params, "training_type", None) == "rigl"


def rigl_params(cfg):
    """(interval, drop_fraction, end_fraction) of a ``training_type: rigl`` config, None for any other config.
    Raises ValueError for an initial ``prune_method`` that is not one-shot, or for out-of-range values."""
    if not is_rigl(cfg):
        return None
    p = cfg.pruning_params
    method = p.prune_method
    if method not in RIGL_INIT_METHODS:
        raise ValueError(f"training_type: rigl needs a one-shot prune_method ({', '.join(RIGL_INIT_METHODS)}) "
                         f"for its initial mask, not '{method}'")
    interval = int(getattr(p, "rigl_update_interval", 100))
    drop = float(getattr(p, "rigl_drop_fraction", 0.3))
    end = float(getattr(p, "rigl_end_fraction", 0.75))
    if interval < 1:
        raise ValueError(f"rigl_update_interval must be >= 1, not {interval}")
    if not 0.0 <= drop <= 1.0:
        raise ValueError(f"rigl_drop_fraction must lie in [0, 1], not {drop}")
    if not 0.0 <= end <= 1.0:
        raise ValueError(f"rigl_end_fraction must lie in [0, 1], not {end}")
    return interval, drop, end


class RiglSchedule:
    def __init__(self, interval: int, drop_fraction: float, end_fraction: float, total_steps: int):
        self.interval = int(interval)
        self.drop_fraction = float(drop_fraction)
        self.end_fraction = float(end_fraction)
        self.total_steps = int(total_steps)
        self.t_end = math.floor(self.end_fraction * self.total_steps)

    @classmethod
    def from_cfg(cls, cfg, total_steps: int):
        return cls(*rigl_params(cfg), total_steps)

    def is_update(self, t: int) -> bool:
        return t > 0 and t % self.interval == 0 and t < self.t_end

    def update_batches(self):
        return [t for t in range(self.t_end) if self.is_update(t)]

    def fraction(self, t: int) -> float:
        return self.drop_fraction / 2 * (1 + math.cos(math.pi * t / self.t_end))

    def k_per_layer(self, t: int, n_active):
        f = self.fraction(t)
        return [int(math.floor(f * int(n))) for n in n_active]
