"""Test-only restatement of DL4J's learning-rate schedules (org.nd4j.linalg.schedule.ISchedule) on top of the DL4J oracle
(oracle/dl4j_oracle.py) without changing it.

Semantics recalled from DL4J 1.0.0-beta3 (PARITY UNPINNED, like the rest of the oracle; the library's statement is include/b200gan.h,
b2g_lr_schedule).  value(i) in double, i = the updater's iteration count before this update's increment (ITERATION) or the epoch count (EPOCH):
  exponential  initial * gamma^i                     inverse  initial / (1 + gamma*i)^power
  sigmoid      initial / (1 + exp(-gamma*(i - step)))  step     initial * decay_rate^floor(i / step)
  map          the value at the largest key <= i
The updater uses value(i) rounded to fp32 once in place of its constant lr.

`enable(net, {layer name: schedule})` gives one oracle Net schedules: it wraps the net's `apply_update` so that each scheduled layer's
`updater.lr` is set to the fp32 value for the net's current iteration / epoch before the update runs, so the oracle's `fit` and `gan_step`
pick the schedules up unchanged.  The schedules are the dicts gan_deeplearning4j_b200.models builds."""
from __future__ import annotations

import copy
import math
import types

import numpy as np

from helpers import oracle_from_specs as _plain_oracle_from_specs


def value(sched, i) -> float:
    """ISchedule.valueAt in double for the schedule's own counter value i."""
    k, i = sched["schedule"], float(i)
    if k == "exponential":
        return sched["initial"] * math.pow(sched["gamma"], i)
    if k == "inverse":
        return sched["initial"] / math.pow(1.0 + sched["gamma"] * i, sched["power"])
    if k == "sigmoid":
        return sched["initial"] / (1.0 + math.exp(-sched["gamma"] * (i - sched["step"])))
    if k == "step":
        return sched["initial"] * math.pow(sched["decay_rate"], math.floor(i / sched["step"]))
    if k == "map":
        best = None
        for key, v in sched["values"]:
            if key <= i and (best is None or key > best[0]):
                best = (key, v)
        assert best is not None, "a MapSchedule must hold key 0"
        return float(best[1])
    raise ValueError(k)


def lr_at(sched, iteration: int, epoch: int) -> np.float32:
    """The fp32 learning rate of an update at (iteration before the increment, epoch)."""
    return np.float32(value(sched, epoch if sched.get("type", "iteration") == "epoch" else iteration))


def _apply_update(self, mb, grads=None, frozen_from=None):
    for name, sched in self.lr_schedules.items():
        u = self.layer_by_name[name].updater
        u.lr = float(lr_at(sched, self.iteration, self.epoch)) if sched is not None else self.lr_constants[name]
    return self.unscheduled_apply_update(mb, grads, frozen_from)


def enable(net, schedules=None):
    """Gives the oracle Net `net` learning-rate schedules {layer name: schedule dict or None (= the constant lr)} and an epoch counter
    (`net.epoch`, set by the caller like Net.set_epoch); returns net.  Call it after any other apply_update wrapper (gradnorm_ref.enable)."""
    if not hasattr(net, "lr_schedules"):
        net.layer_by_name = {l.name: l for l in net.layers}
        net.lr_constants = {l.name: l.updater.lr for l in net.layers if getattr(l, "updater", None) is not None}
        net.lr_schedules, net.epoch = {}, 0
        net.unscheduled_apply_update = net.apply_update
        net.apply_update = types.MethodType(_apply_update, net)
    for name, sched in (schedules or {}).items():
        net.lr_schedules[name] = sched
    return net


def set_schedule(net, sched, layers):
    """Net.set_lr_schedule(sched, layer) for every layer name in `layers` (sched None = back to the constant lr)."""
    enable(net, {name: sched for name in layers})


def scheduled_layers(specs):
    """{layer name: schedule} for the specs whose updater lr is a schedule (new Adam(ISchedule)), layers with a learning rate only."""
    out = {}
    for s in specs:
        u = s.get("updater") or {}
        if isinstance(u.get("lr"), dict) and s["type"] in ("conv2d", "deconv2d", "dense", "output", "batchnorm") and not s.get("frozen", False) \
                and u["kind"] != "noop":
            out[s["name"]] = u["lr"]
    return out


def constant_specs(specs):
    """The specs with every schedule replaced by the constant lr b2g_layer_desc carries for it (its value at 0)."""
    out = copy.deepcopy(list(specs))
    for s in out:
        u = s.get("updater")
        if u and isinstance(u.get("lr"), dict):
            u["lr"] = value(u["lr"], 0)
    return out


def oracle_from_specs(specs, input_shape, **kw):
    """helpers.oracle_from_specs for specs whose updaters may carry schedules; the schedules are enabled on the returned oracle Net."""
    return enable(_plain_oracle_from_specs(constant_specs(specs), input_shape, **kw), scheduled_layers(specs))
