"""Small helpers with the reference's names (torch_utils/misc.py): assert_shape :48, profiled_function :100, InfiniteSampler :111."""

import contextlib
import functools
import itertools
import warnings

import numpy as np
import torch


def assert_shape(tensor, ref_shape):
    if tensor.ndim != len(ref_shape):
        raise AssertionError(f'Wrong number of dimensions: got {tensor.ndim}, expected {len(ref_shape)}')
    for idx, (size, ref_size) in enumerate(zip(tensor.shape, ref_shape)):
        if ref_size is not None and int(size) != int(ref_size):
            raise AssertionError(f'Wrong size for dimension {idx}: got {size}, expected {ref_size}')


def profiled_function(fn):
    @functools.wraps(fn)
    def decorator(*args, **kwargs):
        with torch.autograd.profiler.record_function(fn.__name__):
            return fn(*args, **kwargs)
    return decorator


@contextlib.contextmanager
def suppress_tracer_warnings():
    flt = ('ignore', None, torch.jit.TracerWarning, None, 0)
    warnings.filters.insert(0, flt)
    try:
        yield
    finally:
        warnings.filters.remove(flt)


class InfiniteSampler(torch.utils.data.Sampler):
    """Loops over the dataset forever (the reference's torch_utils/misc.py:111-145).  All ranks share one stream: a permutation drawn from
    RandomState(seed), read cyclically, where each item read swaps its slot with one of the round(window_size * len) slots ending at it,
    so the order drifts from lap to lap.  Rank r of num_replicas takes the stream's items r, r + num_replicas, ...: the shares are
    disjoint.  With shuffle=False the stream is 0, 1, ..., len - 1 over and over."""

    def __init__(self, dataset, rank=0, num_replicas=1, shuffle=True, seed=0, window_size=0.5):
        if not (len(dataset) > 0 and num_replicas > 0 and 0 <= rank < num_replicas and 0 <= window_size <= 1):
            raise ValueError(f'InfiniteSampler: {len(dataset)} items, rank {rank} of {num_replicas}, window {window_size}')
        super().__init__()
        self.dataset, self.rank, self.num_replicas = dataset, rank, num_replicas
        self.shuffle, self.seed, self.window_size = shuffle, seed, window_size

    def _stream(self):
        n = len(self.dataset)
        perm = np.arange(n)
        if not self.shuffle:
            yield from itertools.cycle(perm)
        rng = np.random.RandomState(self.seed)
        rng.shuffle(perm)
        span = int(np.rint(n * self.window_size))
        for slot in itertools.cycle(range(n)):
            item = perm[slot]
            if span > 1:
                other = (slot - rng.randint(span)) % n
                perm[[slot, other]] = perm[[other, slot]]
            yield item

    def __iter__(self):
        return itertools.islice(self._stream(), self.rank, None, self.num_replicas)


def print_module_summary(module, inputs, max_nesting=3, skip_redundant=True):
    """Run module(*inputs) once and print, for every submodule down to `max_nesting` levels, its parameter and buffer counts and its
    first output's shape and dtype (torch_utils/misc.py:199); returns the outputs.  With skip_redundant, submodules that own no
    parameter or buffer of their own and return a tensor already listed are left out."""
    assert isinstance(module, torch.nn.Module) and not isinstance(module, torch.jit.ScriptModule)
    assert isinstance(inputs, (tuple, list))
    names = {m: n for n, m in module.named_modules()}
    depth = {m: (0 if n == '' else n.count('.') + 1) for m, n in names.items()}
    calls = []

    def hook(mod, _inputs, outputs):
        if depth[mod] <= max_nesting:
            outs = outputs if isinstance(outputs, (tuple, list)) else [outputs]
            calls.append((mod, [t for t in outs if isinstance(t, torch.Tensor)]))

    hooks = [m.register_forward_hook(hook) for m in module.modules()]
    try:
        outputs = module(*inputs)
    finally:
        for h in hooks:
            h.remove()

    seen, rows, totals = set(), [], [0, 0]
    for mod, outs in calls:
        params = [t for t in mod.parameters() if id(t) not in seen]
        bufs = [t for t in mod.buffers() if id(t) not in seen]
        new_outs = [t for t in outs if id(t) not in seen]
        seen |= {id(t) for t in params + bufs + new_outs}
        if skip_redundant and not (params or bufs or new_outs):
            continue
        np_, nb = sum(t.numel() for t in params), sum(t.numel() for t in bufs)
        totals[0] += np_
        totals[1] += nb
        name = '<top-level>' if mod is module else names[mod]
        shape, dtype = (str(list(outs[0].shape)), str(outs[0].dtype).split('.')[-1]) if outs else ('-', '-')
        rows.append([name, str(np_) if np_ else '-', str(nb) if nb else '-', shape, dtype])
    table = [[type(module).__name__, 'Parameters', 'Buffers', 'Output shape', 'Datatype']] + rows + [['Total', str(totals[0]), str(totals[1]), '-', '-']]
    widths = [max(len(r[i]) for r in table) for i in range(5)]
    print()
    for r in table:
        print('  '.join(c.ljust(w) for c, w in zip(r, widths)))
    print()
    return outputs
