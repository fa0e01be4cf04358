"""Whole training steps captured in CUDA graphs: one replay = one `train_step` of SupervisedGraphsage,
UnsupervisedGraphsage or Node2VecModel - sampling, the forward and backward kernels, the weight-gradient GEMMs, the clip
to +-5 and Adam (or Node2Vec's four launches) - with no per-kernel host work and no host synchronisation.

    step = model.graphed_train_step(batch_size)
    loss = step(batch, labels)          # supervised; step(batch1, batch2) for the unsupervised and Node2Vec models

RNG contract: replay r draws exactly what the eager train_step would draw at that point of the model's sequence
(neighbour samples, negatives, dropout masks), and eager steps may be interleaved with replays (the short last batch of
an epoch runs eagerly).  The captured kernels read their call counters from device words (the samplers' counter_dev, the
dropout sites' call_dev); before each replay those words are set from the host counters, which then advance by the
step's increments, as an eager step advances them.

Creating a runner switches the model's Adam to capturable=True (step count on the device); from then on the eager
train_step runs that same update, so eager and graphed steps are bit-identical.  Models that never create a runner keep
the default optimiser.
"""
import torch

from . import ops


def make_adam_capturable(optimizer):
    """Switch a live torch.optim.Adam to capturable=True: the step count moves to the parameter's device, so optimizer.step()
    can be captured.  Eager steps then run the capturable update too (its arithmetic differs from the default's in the
    last bits, so compare graphed runs with eager runs of a capturable optimiser)."""
    for group in optimizer.param_groups:
        group["capturable"] = True
        for p in group["params"]:
            st = optimizer.state.get(p)
            if st and "step" in st and st["step"].device != p.device:
                st["step"] = st["step"].to(p.device)
    # eager steps of a capturable optimiser are intended here: skip torch's one-time warning about them
    optimizer._warned_capturable_if_run_uncaptured = True
    return optimizer


class GraphedTrainStep(object):
    """model.train_step for a fixed batch size captured into one CUDA graph (see the module docstring).

    Inputs are copied into static device buffers (non-blocking); the returned loss is a static 0-d CUDA tensor that the
    next replay overwrites (clone it to keep it).  Refused: distributed=True (the gradient all-reduce is not captured),
    layer_infos with different sampler objects, and a batch whose size differs from the captured one."""

    def __init__(self, model, batch_size, warmup=2):
        self.model, self.batch_size = model, int(batch_size)
        if self.batch_size < 1:
            raise ValueError("batch_size must be >= 1")
        if getattr(model, "distributed", False):
            raise NotImplementedError("graphed_train_step with distributed=True is not implemented: the gradient all-reduce "
                                      "(NCCL) is not captured")
        dev = model.device
        # (object, host counter attribute, device offset attribute) of every RNG stream the step draws from
        self.streams = []
        if hasattr(model, "layer_infos"):
            samplers = []
            for info in model.layer_infos:
                if all(info.neigh_sampler is not s for s in samplers):
                    samplers.append(info.neigh_sampler)
            if len(samplers) != 1:
                # one device offset per sampler object would be needed; refuse rather than mis-count (as GraphedForward)
                raise NotImplementedError("graphed_train_step needs all layer_infos to share one neigh_sampler object")
            self.streams.append((samplers[0], "counter", "counter_dev"))
            if model.dropout_rate:
                self.streams.append((model, "dropout_counter", "dropout_call_dev"))
            self.params = model.parameters()
        else:                                                   # Node2VecModel: the two tables (bias in the context table)
            self.params = [model._target, model._context]
        if getattr(model, "neg_sampler", None) is not None:
            self.streams.append((model.neg_sampler, "counter", "counter_dev"))
        B = self.batch_size
        self.inputs = [torch.zeros((B,), dtype=torch.int32, device=dev)]
        if hasattr(model, "num_classes"):                       # supervised: (batch, labels)
            self.inputs.append(torch.zeros((B, model.num_classes), dtype=torch.float32, device=dev))
        else:                                                   # (batch1, batch2)
            self.inputs.append(torch.zeros((B,), dtype=torch.int32, device=dev))
        optimizer = getattr(model, "optimizer", None)
        if optimizer is not None:
            make_adam_capturable(optimizer)
        self.offsets = torch.zeros((max(len(self.streams), 1),), dtype=torch.int64, device=dev)
        self.slots = [self.offsets[i:i + 1] for i in range(len(self.streams))]

        self.stream = torch.cuda.Stream(device=dev)
        self.stream.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(self.stream):
            host0 = [getattr(o, a) for o, a, _ in self.streams]
            saved = self._snapshot(optimizer)
            # warm-up (lazy allocations, cuBLAS handles, Adam's state); its updates and draws are undone below
            model.train_step(*self.inputs)
            self.increments = [getattr(o, a) - h for (o, a, _), h in zip(self.streams, host0)]
            for _ in range(max(int(warmup), 1) - 1):
                model.train_step(*self.inputs)
            self._restore(optimizer, saved)
            self.graph = torch.cuda.CUDAGraph()
            for (o, a, d), slot in zip(self.streams, self.slots):
                setattr(o, a, 0)                                # the graph bakes offsets within the step; the slot adds the base
                setattr(o, d, slot)
            ops.REPACK_ALWAYS[0] = True
            try:
                self.graph.capture_begin(pool=torch.cuda.graph_pool_handle())
                try:
                    self.loss = model.train_step(*self.inputs)
                finally:
                    self.graph.capture_end()
            finally:
                ops.REPACK_ALWAYS[0] = False
                for (o, a, d), h in zip(self.streams, host0):
                    setattr(o, a, h)
                    setattr(o, d, None)                         # eager calls keep the host-numbered sequence
        torch.cuda.current_stream(dev).wait_stream(self.stream)
        ops.CACHE_EPOCH[0] += 1                                 # the restore changed the weights behind the caches' keys
        # what the step leaves on the model for mrr() (the affinities), last_predictions() (the logits) and neg_samples:
        # the graph's tensors, re-bound after every replay because an eager step in between binds its own
        self.bound = {k: getattr(model, k) for k in ("_last", "_last_logits", "neg_samples")
                      if getattr(model, k, None) is not None}
        self.replays = 0

    def _snapshot(self, optimizer):
        params = [p.detach().clone() for p in self.params]
        state = {}
        if optimizer is not None:
            for p in self.params:
                st = optimizer.state.get(p)
                if st:
                    state[p] = {k: v.clone() for k, v in st.items() if torch.is_tensor(v)}
        return params, state

    def _restore(self, optimizer, saved):
        params, state = saved
        with torch.no_grad():
            for p, v in zip(self.params, params):
                p.copy_(v)
            if optimizer is not None:
                for p in self.params:
                    old = state.get(p)
                    for k, v in optimizer.state.get(p, {}).items():
                        if torch.is_tensor(v):
                            if old is None:                     # state the warm-up created: Adam's fresh state is all zeros
                                v.zero_()
                            else:
                                v.copy_(old[k])

    def _load(self, buf, x, name):
        x = torch.as_tensor(x)
        if buf.dim() == 1:
            x = x.reshape(-1)
        if tuple(x.shape) != tuple(buf.shape):
            raise ValueError("graphed_train_step: %s has shape %s, the step was captured for %s (run a batch of another "
                             "size with the eager train_step)" % (name, tuple(x.shape), tuple(buf.shape)))
        buf.copy_(x, non_blocking=True)

    def __call__(self, a, b):
        names = ("batch", "labels") if hasattr(self.model, "num_classes") else ("batch1", "batch2")
        for buf, x, name in zip(self.inputs, (a, b), names):
            self._load(buf, x, name)
        for (o, a_, _), slot, inc in zip(self.streams, self.slots, self.increments):
            h = getattr(o, a_)
            slot.fill_(h)
            setattr(o, a_, h + inc)
        self.graph.replay()
        ops.CACHE_EPOCH[0] += 1                                 # the weights changed without the host seeing it
        for k, v in self.bound.items():
            setattr(self.model, k, v)
        self.replays += 1
        return self.loss
