#!/usr/bin/env python
"""Micro-benchmark of the StyleGAN ops (BASELINE config 5): 512x512x512-channel tensors, achieved GB/s of algorithmic
bytes (numel_in + numel_out)*sizeof(T) against the measured HBM peak.  Prints one JSON line per case.

    python scripts/bench_ops.py [--small]
"""
import argparse, json, os, sys
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ide3d_b200.torch_utils import custom_ops
custom_ops.verbosity = 'none'
from ide3d_b200.torch_utils.ops import bias_act, filtered_lrelu, upfirdn2d


def peak():
    p = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    return float(json.load(open(p))['hbm_gbs']) if os.path.exists(p) else 6650.0


def load_reference_ops():
    """The reference's own torch_utils.ops wrappers on the reference's own CUDA plugins, prebuilt for sm_90a by
    baseline/build_ref_plugins.py (custom_ops._cached_plugins is pre-seeded, so get_plugin returns them without a JIT build)."""
    import importlib.util
    ref = os.path.join(ROOT, 'baseline', '_ref')
    if not os.path.isdir(os.path.join(ref, 'plugins')):
        return None
    sys.path.insert(0, ref)
    from torch_utils import custom_ops as rco
    rco.verbosity = 'none'
    for name in ('bias_act_plugin', 'upfirdn2d_plugin', 'filtered_lrelu_plugin'):
        spec = importlib.util.spec_from_file_location(name, os.path.join(ref, 'plugins', name, name + '.so'))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        rco._cached_plugins[name] = mod
    from torch_utils.ops import bias_act as r_ba, filtered_lrelu as r_fl, upfirdn2d as r_up
    return r_ba, r_fl, r_up


def timeit(fn, reps=10, warm=3):
    flush = torch.empty(256 * 1024 * 1024 // 4, device='cuda')
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); y = fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--small', action='store_true')
    ap.add_argument('--no-ref', action='store_true', help='skip the reference plugins (baseline/_ref)')
    ap.add_argument('--only', default=None, help='substring filter on the op name')
    args = ap.parse_args()
    C = 64 if args.small else 512
    pk = peak()
    f4 = upfirdn2d.setup_filter([1, 3, 3, 1], device='cuda')
    import scipy.signal
    f12 = torch.as_tensor(scipy.signal.firwin(numtaps=12, cutoff=0.25, width=0.5), dtype=torch.float32, device='cuda')
    refops = None if args.no_ref else load_reference_ops()
    for dtype in (torch.float32, torch.float16):
        x = torch.randn(1, C, 512, 512, device='cuda', dtype=dtype)
        b = torch.randn(C, device='cuda', dtype=dtype)
        flkw = dict(fu=f12, fd=f12, b=b, up=2, down=2, padding=[10, 11, 10, 11], gain=2 ** 0.5, slope=0.2, clamp=256)
        cases = {
            'bias_act lrelu+clamp': lambda m: m[0].bias_act(x, b, act='lrelu', clamp=256),
            'upfirdn2d upsample2d 4x4': lambda m: m[2].upsample2d(x, f4),
            'upfirdn2d filter2d 4x4': lambda m: m[2].filter2d(x, f4),
            'upfirdn2d downsample2d 4x4': lambda m: m[2].downsample2d(x, f4),
            'filtered_lrelu up2 down2 12-tap': lambda m: m[1].filtered_lrelu(x, **flkw),
        }
        ours = (bias_act, filtered_lrelu, upfirdn2d)
        for layout in ('contiguous', 'channels_last'):
            if layout == 'channels_last':
                x = x.contiguous(memory_format=torch.channels_last)
            for name, fn in cases.items():
                if args.only and args.only not in name:
                    continue
                try:
                    ms, y = timeit(lambda: fn(ours))
                except Exception as e:          # noqa
                    print(json.dumps({'op': name, 'dtype': str(dtype), 'layout': layout, 'error': str(e)[:200]}))
                    continue
                nbytes = (x.numel() + y.numel()) * x.element_size()
                gbs = nbytes / ms / 1e6
                rec = {'op': name, 'dtype': str(dtype).replace('torch.', ''), 'layout': layout, 'shape': list(x.shape), 'out': list(y.shape),
                       'ours_ms': round(ms, 4), 'algorithmic_GB': round(nbytes / 1e9, 3), 'achieved_GBs': round(gbs, 1), 'peak_GBs': pk, 'frac': round(gbs / pk, 3)}
                if refops is not None:              # the reference's own sm_90a-compiled plugin on the same tensor, same call
                    try:
                        with torch.no_grad():
                            rms, ry = timeit(lambda: fn(refops), reps=5, warm=2)
                        rec.update(ref_plugin_ms=round(rms, 4), speedup_vs_ref_plugin=round(rms / ms, 2),
                                   max_abs_diff_vs_ref_plugin=float((ry.float() - y.float()).abs().max()))
                        del ry
                    except Exception as e:      # noqa
                        rec.update(ref_plugin_error=str(e)[:160])
                print(json.dumps(rec), flush=True)
                del y

    # ---- the fused forms on the shapes of the synthesis step (NHWC fp32, batch 8): algorithmic bytes = every tensor once
    def fused_case(name, fn, nbytes):
        if args.only and args.only not in name:
            return
        try:
            ms, y = timeit(fn)
        except Exception as e:          # noqa
            print(json.dumps({'op': name, 'error': str(e)[:200]}))
            return
        gbs = nbytes / ms / 1e6
        print(json.dumps({'op': name, 'dtype': 'float32', 'layout': 'channels_last', 'ms': round(ms, 4), 'algorithmic_GB': round(nbytes / 1e9, 3),
                          'achieved_GBs': round(gbs, 1), 'peak_GBs': pk, 'frac': round(gbs / pk, 3)}), flush=True)

    cl = lambda t: t.contiguous(memory_format=torch.channels_last)
    n = 2 if args.small else 8
    xt = cl(torch.randn(n, 64, 513, 513, device='cuda'))                       # b512.conv0: transposed-conv output
    d, s2, bb = torch.rand(n, 64, device='cuda') + 0.5, torch.rand(n, 64, device='cuda') + 0.5, torch.randn(64, device='cuda')
    nz = torch.randn(512, 512, device='cuda')
    fused_case('upfirdn2d_epilogue b512.conv0 (FIR + demod + noise + bias + lrelu -> x*s1)',
               lambda: upfirdn2d.upfirdn2d_epilogue(xt, f4, padding=[1, 1, 1, 1], gain=4, scale=d, noise=nz, b=bb, act='lrelu', next_scale=s2, only_next=True),
               (xt.numel() + n * 64 * 512 * 512) * 4)
    xc = cl(torch.randn(n, 64, 512, 512, device='cuda'))                       # b512.conv1 output
    fused_case('scaled_bias_act b512.conv1 (demod + noise + bias + lrelu -> x and x*s_rgb)',
               lambda: bias_act.scaled_bias_act(xc, scale=d, noise=nz, b=bb, act='lrelu', next_scale=s2), 3 * xc.numel() * 4)
    fused_case('scaled_bias_act modulation only (x * styles)', lambda: bias_act.scaled_bias_act(xc, scale=d), 2 * xc.numel() * 4)
    img = cl(torch.randn(n, 96, 128, 128, device='cuda'))                      # vb256 skip step
    ywide = cl(torch.randn(n, 192, 256, 256, device='cuda'))
    b96 = torch.randn(96, device='cuda')
    fused_case('upsample2d_add vb256 (upsample2d(img) + y[:, :96] + b)', lambda: upfirdn2d.upsample2d_add(img, f4, ywide[:, :96], b96),
               (img.numel() + 2 * n * 96 * 256 * 256) * 4)


if __name__ == '__main__':
    main()
