#!/usr/bin/env python
"""Where the time of one bench step goes, and what folding ToRGB / chaining styles across blocks (networks.FUSED_TORGB) changes.

    python scripts/bench_synthesis_passes.py [--steps 20] [--rounds 3] [--out DIR]

The workload is bench.py's: G.synthesis for 8 latents of the random-init bench generator, 64^2 x 96 render -> 512^2.
1. profile  : one step per path under torch.profiler (CUDA activities, a run of its own after the timing): ms and launches per
              kernel name, grouped as ray-march / this project's elementwise + FIR kernels / cuDNN 1x1 / other cuDNN convolutions
              (attributed through the aten convolution op and its weight shape) / other; plus the bytes the elementwise
              epilogues stream (inputs + outputs of every bias_act / modconv_epilogue(_rgb) call, counted from the shapes).
2. timing   : steps with the switch off and on, alternating in one process for --rounds rounds (CUDA events, L2 flushed between
              steps as in bench.py).
3. results  : max |image(on) - image(off)| once with fp32 convolutions (cudnn.allow_tf32 = False) and once as benched.
The card's name and power limit are read in the same run.  Prints one JSON document (also written to DIR/synthesis_passes.json).
"""

import argparse
import collections
import json
import os
import re
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GROUPS = (('ray-march', re.compile(r'raymarch')),
          ('ours: elementwise / FIR', re.compile(r'modconv_epilogue|upfirdn2d|bias_act')))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [v.strip() for v in q.split(',')]
        return {'name': name, 'power_limit': power, 'max_sm_clock': clock}
    except Exception as e:                     # noqa: BLE001 -- the numbers are still valid, only unlabelled
        return {'name': torch.cuda.get_device_name(), 'power_limit': f'unknown ({e})'}


class ByteCounter:
    """Counts the bytes every elementwise epilogue call reads (x) and writes (its outputs), from the tensor shapes."""

    def __init__(self):
        from ide3d_b200 import _plugins
        self.plugin = _plugins.PLUGINS['bias_act_plugin']
        self.saved = {k: getattr(self.plugin, k) for k in ('bias_act', 'modconv_epilogue', 'modconv_epilogue_rgb')}
        self.bytes = 0
        self.calls = 0

    def __enter__(self):
        def wrap(fn):
            def counted(x, *a, **k):
                out = fn(x, *a, **k)
                if out is not None:
                    outs = out if isinstance(out, (list, tuple)) else [out]
                    self.bytes += x.numel() * x.element_size() + sum(t.numel() * t.element_size() for t in outs)
                    self.calls += 1
                return out
            return counted
        for k, fn in self.saved.items():
            setattr(self.plugin, k, wrap(fn))
        return self

    def __exit__(self, *exc):
        for k, fn in self.saved.items():
            setattr(self.plugin, k, fn)


def profile_step(step):
    from torch.profiler import ProfilerActivity, profile
    step()
    torch.cuda.synchronize()
    with ByteCounter() as bc, profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], record_shapes=True) as prof:
        step()
        torch.cuda.synchronize()
    events = prof.events()
    per_name = collections.defaultdict(lambda: [0, 0.0])
    for e in events:
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = re.sub(r'\(.*', '', e.name)[:110]
            per_name[name][0] += 1
            per_name[name][1] += e.time_range.elapsed_us() / 1e3
    conv = {'cuDNN 1x1 convolutions': [0, 0.0], 'cuDNN 3x3 / transposed convolutions': [0, 0.0]}
    for e in events:
        if e.device_type == torch.autograd.DeviceType.CPU and e.name in ('aten::cudnn_convolution', 'aten::cudnn_convolution_transpose') and e.kernels:
            wshape = e.input_shapes[1] if len(e.input_shapes) > 1 else []
            key = 'cuDNN 1x1 convolutions' if (e.name == 'aten::cudnn_convolution' and len(wshape) == 4 and wshape[2:] == [1, 1]) \
                else 'cuDNN 3x3 / transposed convolutions'
            conv[key][0] += len(e.kernels)
            conv[key][1] += sum(k.duration for k in e.kernels) / 1e3
    groups = collections.OrderedDict((g, [0, 0.0]) for g, _ in GROUPS)
    total = [0, 0.0]
    for name, (n, ms) in per_name.items():
        total[0] += n
        total[1] += ms
        for g, rx in GROUPS:
            if rx.search(name):
                groups[g][0] += n
                groups[g][1] += ms
                break
    groups.update(conv)
    groups['other'] = [total[0] - sum(v[0] for v in groups.values()), total[1] - sum(v[1] for v in groups.values())]
    top = sorted(per_name.items(), key=lambda kv: -kv[1][1])[:25]
    return {'kernel_ms_total': round(total[1], 3), 'launches': total[0],
            'groups': {g: {'ms': round(ms, 3), 'launches': n, 'share': round(ms / total[1], 3)} for g, (n, ms) in groups.items()},
            'epilogue_bytes': bc.bytes, 'epilogue_calls': bc.calls,
            'kernels': [{'name': k, 'launches': n, 'ms': round(ms, 3)} for k, (n, ms) in top]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this measurement needs a CUDA device'
    from bench import BATCH, NUM_STEPS, build_generator, make_labels, make_latents
    from ide3d_b200.training import networks as nw

    dev = torch.device('cuda:0')
    torch.backends.cudnn.benchmark = True
    G = build_generator(dev)
    with torch.no_grad():
        ws = G.mapping(make_latents(BATCH, G.z_dim).to(dev), make_labels(BATCH).to(dev))
    c = make_labels(BATCH).to(dev)
    kw = dict(render_params=dict(num_steps=NUM_STEPS), noise_mode='const', perturb='hash', seed=1)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    saved = nw.FUSED_TORGB

    def run(fused):
        nw.FUSED_TORGB = fused
        return G.synthesis(ws, c=c, **kw)

    report = {'card': card(), 'workload': 'G.synthesis, 8 latents, 64^2 x 96 -> 512^2 (bench.py)'}
    try:
        with torch.no_grad():
            for fused in (False, True):                        # warm both paths (cuDNN algorithm choice, module loads)
                for _ in range(3):
                    run(fused)
            torch.cuda.synchronize()
            rounds = {False: [], True: []}
            for _ in range(args.rounds):
                for fused in (False, True):
                    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
                    for a, b in ev:
                        flush.zero_()
                        a.record()
                        run(fused)
                        b.record()
                    torch.cuda.synchronize()
                    rounds[fused].append(float(np.mean([a.elapsed_time(b) for a, b in ev])))
            report['timing_ms_per_step'] = {'fused_off': [round(v, 3) for v in rounds[False]], 'fused_on': [round(v, 3) for v in rounds[True]],
                                            'steps_per_round': args.steps}
            diffs = {}
            for label, tf32 in (('fp32_convolutions', False), ('as_benched', True)):
                prev = torch.backends.cudnn.allow_tf32
                torch.backends.cudnn.allow_tf32 = tf32
                try:
                    a, b = run(False).float(), run(True).float()
                finally:
                    torch.backends.cudnn.allow_tf32 = prev
                diffs[label] = {'max_abs_diff': (a - b).abs().max().item(), 'max_abs_ref': a.abs().max().item()}
                diffs[label]['relative'] = diffs[label]['max_abs_diff'] / max(diffs[label]['max_abs_ref'], 1e-30)
            report['image_diff'] = diffs
            report['profile'] = {'fused_off': profile_step(lambda: run(False)), 'fused_on': profile_step(lambda: run(True))}
    finally:
        nw.FUSED_TORGB = saved
    text = json.dumps(report, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'synthesis_passes.json'), 'w') as f:
            f.write(text)


if __name__ == '__main__':
    main()
