"""What the two trainers (supervised_train.py, unsupervised_train.py) share: tf.app.flags-style command lines, the --gpu
device choice, the reference's epoch loop, the time= clock and the host -> device copies of a batch.

Flags are spelled as the reference's scripts spell them: `--name value`, `--name=value`, and for booleans `--name`,
`--noname` or `--name=true|false`.  An unknown flag or a stray argument is an error."""
import time
import types

import numpy as np
import torch


class FlagError(ValueError):
    pass


_TRUE, _FALSE = ("true", "t", "1"), ("false", "f", "0")
_CONVERT = {"integer": int, "float": float, "string": str}


def parse_flags(spec, argv):
    """spec: [(name, kind, default)] with kind "boolean" / "integer" / "float" / "string" (tf.app.flags.DEFINE_<kind>).
    Returns a namespace with one attribute per flag."""
    kinds = {name: kind for name, kind, _ in spec}
    values = {name: default for name, _, default in spec}
    argv = list(argv)
    i = 0
    while i < len(argv):
        tok = argv[i]
        i += 1
        if not tok.startswith("-") or tok.strip("-") == "":
            raise FlagError("unexpected argument %r" % (tok,))
        name, eq, value = tok.lstrip("-").partition("=")
        if name not in kinds and name.startswith("no") and kinds.get(name[2:]) == "boolean" and not eq:
            values[name[2:]] = False
            continue
        if name not in kinds:
            raise FlagError("unknown flag --%s" % name)
        kind = kinds[name]
        if kind == "boolean":
            if not eq or value.lower() in _TRUE:
                values[name] = True
            elif value.lower() in _FALSE:
                values[name] = False
            else:
                raise FlagError("flag --%s: %r is not a boolean" % (name, value))
            continue
        if not eq:
            if i >= len(argv):
                raise FlagError("flag --%s needs a value" % name)
            value = argv[i]
            i += 1
        try:
            values[name] = _CONVERT[kind](value)
        except ValueError:
            raise FlagError("flag --%s: %r is not a valid %s" % (name, value, kind))
    return types.SimpleNamespace(**values)


def parse_or_exit(spec, argv):
    try:
        return parse_flags(spec, argv)
    except FlagError as e:
        raise SystemExit("error: %s" % e)


def select_device(gpu):
    """cuda:<gpu>, or cuda:0 (with one line of output) when that device does not exist.  CUDA_VISIBLE_DEVICES is left
    alone: the reference's default --gpu 1 would hide the only GPU of a one-GPU machine, and there is no CPU path."""
    if not torch.cuda.is_available():
        raise RuntimeError("the trainers need a CUDA device (there is no CPU fallback)")
    n = torch.cuda.device_count()
    if not 0 <= gpu < n:
        print("--gpu %d: no such device (%d visible), using cuda:0" % (gpu, n))
        gpu = 0
    device = torch.device("cuda", gpu)
    torch.cuda.set_device(device)
    return device


def to_device(x, dtype, device):
    """Host array -> device tensor through pinned memory, without blocking the host."""
    host = torch.from_numpy(np.ascontiguousarray(x, dtype=dtype))
    return host.pin_memory().to(device, non_blocking=True)


class StepClock(object):
    """time=: the reference averages the wall time of synchronous sess.run calls.  A step here returns before the GPU has
    finished it, so the clock runs from the first step and every reading ends with a device synchronise; avg() is the
    wall time so far per step (host iterator and validations included, as they fall between the readings)."""

    def __init__(self, device, sync=None):
        self.sync = sync if sync is not None else (lambda: torch.cuda.synchronize(device))
        self.t0 = time.time()

    def avg(self, steps):
        self.sync()
        return (time.time() - self.t0) / steps


def train_loop(minibatch, flags, step, validate, after):
    """The epoch loop of the reference (supervised_train.py:262-312, unsupervised_train.py:260-316).

    step(item, iter, total_steps, eager) runs the training step on item = next_minibatch_feed_dict(); eager is True on
    print steps (they read the step's outputs) and for a batch shorter than flags.batch_size, else the step may be a
    graph replay.  validate() runs when iter % validate_iter == 0 and returns the validation cost; after(out, iter,
    total_steps, printing) follows every step (printing on total_steps % print_every == 0).  Returns (total_steps,
    epoch_val_costs)."""
    total_steps = 0
    epoch_val_costs = []
    for epoch in range(flags.epochs):
        minibatch.shuffle()
        it = 0
        print('Epoch: %04d' % (epoch + 1))
        epoch_val_costs.append(0)
        while not minibatch.end():
            item = minibatch.next_minibatch_feed_dict()
            feed = item[0] if isinstance(item, tuple) else item
            printing = total_steps % flags.print_every == 0
            out = step(item, it, total_steps, printing or feed["batch_size"] != flags.batch_size)
            if it % flags.validate_iter == 0:
                epoch_val_costs[-1] += validate()
            after(out, it, total_steps, printing)
            it += 1
            total_steps += 1
            if total_steps > flags.max_total_steps:
                break
        if total_steps > flags.max_total_steps:
            break
    return total_steps, epoch_val_costs
