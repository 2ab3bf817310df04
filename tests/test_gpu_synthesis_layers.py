"""Every synthesis layer of the benchmark's step against float64, one layer at a time, with bias and noise switched on.

The generator is the one bench.py times (compat.random_init_generator(seed=0), batch 8, bench.make_latents / make_labels,
noise_mode='const'), so cuDNN and this package's kernels see the launch geometry of the benchmark: the 512-channel TMA FIR tiles,
the 192-channel backbone ToRGB, `epilogue_rgb` at 128 and 64 channels on 256^2 and 512^2.  Random init has zero biases and zero
noise strengths, which would let every epilogue add zeros; switch_on_terms() gives each layer a distinct noise strength, each conv /
ToRGB bias N(0, 0.1^2) values and each affine bias 0.3 N(0, 1) on top of its 1, so styles vary per channel.

SynthesisLayer / ToRGBLayer / SynthesisBlock / SegSynthesisBlock.forward are wrapped (LayerChecker).  Each wrapper keeps the first and
the last sample of the batch (every stage is per-sample), calls the original, and checks what the call returned against a float64
reference computed on the device FROM THAT CALL'S OWN INPUTS -- errors do not compound, each stage is judged alone.  Styles and
demodulation coefficients are recomputed in float64 from the ws rows.  The float64 tensors of a call are freed before the next call;
their peak (printed) was 3.25 GiB on an H100 80GB HBM3 (700 W power limit), where the whole file ran in 39 s.

Bounds are per element and follow from the operand formats (u = 2^-24, gamma_k = k u / (1 - k u)); nothing in them is fitted:
- styles: gamma_(K+4) (sum_k |A w| + |b|) for a K-term float32 affine; dcoefs: the float32 sum of squares (gamma_(I+12)) plus the
  styles' error, through rsqrt (relative error <= half that of its argument, at most 2 ulp for rsqrtf).
- convolution, relative to A = conv(|x|, |W|) (through |f| for conv0), K = I k^2 products: float32 gamma_K; TF32 (the SR blocks under
  allow_tf32) 2 2^-10 + gamma_K, each operand rounded or truncated to 10 bits; fp16 operands (the backbone under allow_tf32)
  gamma_K plus the fp16 weight copy W 2^-e, max(2^-11 |W|, 2^-25 2^e) per weight (2^-25 for weights below fp16's normal range), plus
  the fp16 rounding of the convolution output, 2^-11 |c| + 2^-25 2^e.  conv0's raw output is bounded through the FIR with |f| (its
  16-tap float32 sum adds gamma_16).
- tail: x d + noise + b (three roundings), lrelu (slope <= 1) times sqrt(2) (three more), times the next styles (one more), each
  carrying the error of its operands; 2^-11 |v| + 2^-25 where the output is fp16.  Folded ToRGB: gamma_(C+3) on the C-term sum.
- skip: upsample2d(img) + y + b, gamma_8 over upsample2d(|img|) + |y| + |b|.
cuDNN is left to pick its algorithms as the benchmark does (cudnn.benchmark on); the bounds above assume a product-summing algorithm
(implicit GEMM, direct).  A Winograd or FFT pick would need its own constant, and a change of pick shows here first as a failure.

Negative controls: five realistic defects are applied to copies of captured kernel outputs (noise shifted by one pixel, one 4-channel
bias vector dropped, next styles taken from the other sample, one edge row of a 16 x 16 FIR tile zeroed, the last row of a skip image
not upsampled); each must break the bound somewhere.  test_layer_checker_rehearsal_on_cpu runs the same capture, reference, bounds and
controls on a reduced generator under the CPU oracle, where the blocks take the unfolded NCHW forms."""

import time

import pytest
import torch
import torch.nn.functional as F

from oracle import ops as oops

U32, H16, SUB16 = 2.0 ** -24, 2.0 ** -11, 2.0 ** -25
F16_MAX = 65504.0


def gamma(k):
    return k * U32 / (1 - k * U32)


def switch_on_terms(G, seed=1):
    """Non-zero noise strengths (0.1 |N(0,1)|, one per layer), conv / ToRGB biases N(0, 0.1^2), affine biases + 0.3 N(0,1)."""
    from ide3d_b200.training import networks, triplane
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in G.synthesis.modules():
            if isinstance(m, (networks.SynthesisLayer, networks.ToRGBLayer)):
                if getattr(m, 'use_noise', False):
                    m.noise_strength.copy_(0.1 * torch.randn([], generator=g).abs())
                m.bias.copy_(0.1 * torch.randn(m.bias.shape, generator=g))
                m.affine.bias.add_(0.3 * torch.randn(m.affine.bias.shape, generator=g).to(m.affine.bias.device))
    triplane.invalidate_caches(G)
    return G


def blocks_of(synthesis):
    """[(chain name, [blocks])]: the backbone and the SR head, each a chain of blocks linked by their epilogues."""
    return [('backbone', [getattr(synthesis, f'vb{r}') for r in synthesis.voxel_block_resolutions]),
            ('sr', [getattr(synthesis, f'b{r}') for r in synthesis.block_resolutions])]


def ws_rows(synthesis):
    """{layer: index of its ws row} -- the rule of split_ws / StylePlan: conv0, conv1, torgb; the base advances by num_conv."""
    rows, idx = {}, 0
    for _, blocks in blocks_of(synthesis):
        for b in blocks:
            j = idx
            if b.in_channels != 0:
                rows[b.conv0] = j
                j += 1
            rows[b.conv1] = j
            rows[b.torgb] = j + 1
            idx += b.num_conv
    return rows


# ------------------------------------------------------------------------------------------------ float64 reference + bounds
def style_ref(layer, w):
    """float64 styles of `layer` from ws rows w [n, w_dim] (float32 values), and their bound for a float32 evaluation."""
    from ide3d_b200.training import networks
    aff = layer.affine
    A = aff.weight.double() * aff.weight_gain
    b = aff.bias.double() * aff.bias_gain
    out = float(layer.weight_gain) if isinstance(layer, networks.ToRGBLayer) else 1.0
    w = w.double()
    s = (w @ A.t() + b) * out
    es = gamma(w.shape[1] + 4) * (w.abs() @ A.abs().t() + b.abs()) * out
    return s, es


def demod_ref(layer, s, es):
    """float64 rsqrt(sum_i s_i^2 sum_k W_oik^2 + 1e-8) and its bound, given styles s with bound es."""
    W = layer.weight.double().contiguous()
    Q = W.square().sum(dim=[2, 3])
    S = s.square() @ Q.t() + 1e-8
    dS = ((2 * s.abs() + es) * es) @ Q.t() * (1 + gamma(10)) + gamma(W.shape[1] + 12) * S
    rel = dS / S
    assert float(rel.max()) < 0.5
    d = S.rsqrt()
    return d, d * (rel + 5 * U32)


def _cv(t):                     # [n, C] -> [n, C, 1, 1]
    return t[:, :, None, None]


def tail(c, d, nz, b, gain):
    v = c * _cv(d) + nz + b[None, :, None, None]
    return gain * torch.where(v >= 0, v, 0.2 * v)


def tail_bound(c, ec, d, ed, nz, b, gain):
    """Bound on the tail's output given |c~ - c| <= ec and |d~ - d| <= ed: fma + noise rounding + bias add, then lrelu * gain."""
    chi, dhi = c.abs() + ec, _cv(d.abs() + ed)
    e_pre = ec * dhi + chi * _cv(ed) + gamma(3) * (chi * dhi + nz.abs() + b.abs()[None, :, None, None]) + U32 * nz.abs()
    y = tail(c, d, nz, b, gain)
    return y, gain * e_pre + gamma(3) * (y.abs() + gain * e_pre)


def conv_weight_bound(W, k, mode, e=0):
    """Per-weight factor B with |c~ - c| <= conv(|x|, B): mode 'fp32' | 'tf32' | 'fp16' (weight copy W 2^-e rounded to fp16)."""
    a = W.abs()
    if mode == 'fp16':
        dw = torch.clamp(H16 * a, min=SUB16 * 2.0 ** e)
        return gamma(k) * (a + dw) + dw
    if mode == 'tf32':
        return (2 * 2.0 ** -10 + 2.0 ** -20 + gamma(k) * (1 + 2.0 ** -10) ** 2) * a
    return gamma(k) * a


class LayerChecker:
    """Wraps the layer and block forwards (install), checks each call as it returns, records one line per call.

    samples: batch indices kept (first and last).  controls: {defect: stage name} for the negative controls.  After the run:
    self.lines (per call: stage, shape, dtype, max err / bound, fp16 headroom max|v| / 65504), self.events (the call sequence with
    the form of each output), self.rejected {defect: max err / bound of the defective output, > 1 when rejected}, self.peak (largest extra device memory of one check, bytes)."""

    def __init__(self, G, ws, samples, controls, verbose=True):
        from ide3d_b200.training import networks
        self.nw = networks
        self.syn = G.synthesis
        self.samples = list(samples)
        self.ws = ws[self.samples].detach().clone()
        self.rows = ws_rows(self.syn)
        self.names = {m: n for n, m in self.syn.named_modules()}
        self.chain_next = {}                     # block -> next block of its chain
        for _, blocks in blocks_of(self.syn):
            for a, b in zip(blocks, blocks[1:]):
                self.chain_next[a] = b
        self.block_of = {m: b for _, blocks in blocks_of(self.syn) for b in blocks for m in (b.conv1, b.torgb) + ((b.conv0,) if b.in_channels else ())}
        self.controls = dict(controls)
        self.rejected = {}
        self.lines, self.events, self.calls = [], [], []
        self.block_rgb = {}
        self.peak = 0
        self.verbose = verbose
        self._styles = {}

    # ---- helpers
    def styles(self, layer):
        if layer not in self._styles:
            self._styles[layer] = style_ref(layer, self.ws[:, self.rows[layer]])
        return self._styles[layer]

    def _pick(self, t):
        return None if t is None else t[self.samples].detach().contiguous()

    def _conv_mode(self, x, fp16):
        if fp16:
            return 'fp16'
        return 'tf32' if x.is_cuda and bool(torch.backends.cudnn.allow_tf32) else 'fp32'

    def _record(self, stage, kind, out, ref, bound):
        out64 = out.double()
        err = (out64 - ref).abs()
        ratio = float((err / bound).max())
        head = None
        if out.dtype == torch.float16:
            assert bool(torch.isfinite(out).all()), f'{stage}: non-finite fp16 values'
            head = float(out.float().abs().max()) / F16_MAX
        bad = err > bound
        line = dict(stage=stage, kind=kind, shape=tuple(out.shape), dtype=str(out.dtype).replace('torch.', ''), ratio=ratio, headroom=head)
        self.lines.append(line)
        if self.verbose:
            print(f"{stage:>14s} {kind:<6s} {str(line['shape']):<22s} {line['dtype']:<8s} max err/bound {ratio:.3f}"
                  + ('' if head is None else f'  fp16 max|v|/65504 {head:.2e}'))
        assert not bool(bad.any()), (f'{stage} {kind}: {int(bad.sum())} / {bad.numel()} elements over the bound, '
                                     f'max err/bound {ratio:.3g}')

    def _control(self, defect, stage, out, ref, ref_defect, bound):
        """A defect moves the kernel's output by ref_defect - ref; the check must reject it somewhere."""
        if self.controls.get(defect) != stage:
            return
        bad = (out.double() + (ref_defect - ref)).to(out.dtype).double()
        self.rejected[defect] = float(((bad - ref).abs() / bound).max())      # rejected when > 1

    def _begin(self):
        if torch.cuda.is_available():
            torch.cuda.synchronize()
            self._m0 = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()

    def _end(self):
        if torch.cuda.is_available():
            torch.cuda.synchronize()
            self.peak = max(self.peak, torch.cuda.max_memory_allocated() - self._m0)

    # ---- the wrapped forwards
    def install(self, monkeypatch):
        nw = self.nw
        orig = {cls: cls.forward for cls in (nw.SynthesisLayer, nw.ToRGBLayer, nw.SynthesisBlock, nw.SegSynthesisBlock)}
        chk = self

        def layer_fwd(layer, x, w, **kw):
            cap = dict(x=chk._pick(x), kw={k: v for k, v in kw.items() if k not in ('styles', 'dcoefs', 'next_styles', 'y_styles', 'rgb')},
                       styles=chk._pick(kw.get('styles')), dcoefs=chk._pick(kw.get('dcoefs')), next_styles=chk._pick(kw.get('next_styles')),
                       y_styles=chk._pick(kw.get('y_styles')), rgb=None if kw.get('rgb') is None else (kw['rgb'][0], chk._pick(kw['rgb'][1]), kw['rgb'][2]))
            out = orig[nw.SynthesisLayer](layer, x, w, **kw)
            chk.check_layer(layer, cap, out)
            return out

        def torgb_fwd(layer, x, w, **kw):
            cap = dict(x=chk._pick(x), premodulated=kw.get('premodulated', False), raw=kw.get('raw', False))
            out = orig[nw.ToRGBLayer](layer, x, w, **kw)
            chk.check_torgb(layer, cap, out)
            return out

        def block_fwd(block, x, img, ws, **kw):
            cap = dict(img=chk._pick(img))
            chk.events.append((chk.names[block], 'enter'))
            out = orig[nw.SynthesisBlock](block, x, img, ws, **kw)
            chk.check_skip(block, [(cap['img'], out[1], slice(None))])
            return out

        def seg_block_fwd(block, x, img, ws, condition_img=None, **kw):
            cap = dict(img=chk._pick(img), seg=chk._pick(condition_img))
            chk.events.append((chk.names[block], 'enter'))
            out = orig[nw.SegSynthesisBlock](block, x, img, ws, condition_img=condition_img, **kw)
            ci = block.img_channels
            chk.check_skip(block, [(cap['img'], out[1], slice(0, ci)), (cap['seg'], out[2], slice(ci, None))])
            return out

        monkeypatch.setattr(nw.SynthesisLayer, 'forward', layer_fwd)
        monkeypatch.setattr(nw.ToRGBLayer, 'forward', torgb_fwd)
        monkeypatch.setattr(nw.SynthesisBlock, 'forward', block_fwd)
        monkeypatch.setattr(nw.SegSynthesisBlock, 'forward', seg_block_fwd)

    # ---- the checks
    def check_layer(self, layer, cap, out):
        self._begin()
        name = self.names[layer]
        block = self.block_of[layer]
        kw = cap['kw']
        assert kw.get('noise_mode') == 'const' and kw.get('fused_modconv') is False and layer.conv_clamp is None, name
        outs = [out] if isinstance(out, torch.Tensor) else list(out)
        kinds = []
        if kw.get('emit_y', True) and not kw.get('only_next', False):
            kinds.append('y*ys' if cap['y_styles'] is not None else 'y')
        if cap['next_styles'] is not None:
            kinds.append('y*sn')
        if cap['rgb'] is not None:
            kinds.append('rgb')
        assert len(outs) == len(kinds), (name, len(outs), kinds)
        self.events.append((name, tuple(kinds)))
        fp16 = bool(kw.get('fp16', False))
        e = layer.fp16_exponent() if fp16 else 0
        self.calls.append(dict(stage=name, x=cap['x'].dtype, outs=tuple(o.dtype for o in outs), fp16=fp16))

        # styles and demodulation in float64 from the ws row; the passed ones must sit inside their bounds
        s, es = self.styles(layer)
        d, ed = demod_ref(layer, s, es)
        if cap['styles'] is not None:
            assert bool(((cap['styles'].double() - s).abs() <= es).all()), f'{name}: styles'
        if cap['dcoefs'] is not None:
            assert bool(((cap['dcoefs'].double() - d * 2.0 ** e).abs() <= ed * 2.0 ** e).all()), f'{name}: dcoefs'

        # the convolution input: premodulated x as it arrives, else x * s formed inside the layer
        x = cap['x']
        if kw.get('premodulated', False):
            xm = x.double()
            e_in = None
        else:
            x64 = x.double()
            xm = x64 * _cv(s)
            e_in = x64.abs() * _cv(es)
            e_in = e_in + (H16 * (xm.abs() + e_in) + SUB16 if fp16 else U32 * (xm.abs() + e_in))
        x_abs = xm.abs() if e_in is None else xm.abs() + e_in
        W = layer.weight.double().contiguous()
        mode = self._conv_mode(x, fp16)
        K = W.shape[1] * W.shape[2] * W.shape[3]
        Wb = conv_weight_bound(W, K, mode, e)
        f = layer.resample_filter.double()
        if layer.up > 1:
            conv = lambda t, w: oops.conv2d_resample(t, w, f=f, up=2, padding=layer.padding, flip_weight=False)
            c = conv(xm, W)
            ec = conv(x_abs, Wb)
            if e_in is not None:
                ec = ec + conv(e_in, W.abs())
            # the transposed convolution's own output, through the FIR with |f| (f >= 0): its rounding and the FIR's 16-term sum
            raw = oops.upfirdn2d(F.conv_transpose2d(xm, W.transpose(0, 1), stride=2).abs(), f, padding=1, gain=4)
            assert raw.shape == c.shape and bool((raw >= c.abs() * (1 - 1e-9)).all()), f'{name}: FIR magnitude'
            raw_hi = raw + ec
            ec = ec + (H16 * raw_hi + 4 * SUB16 * 2.0 ** e if fp16 else U32 * raw_hi) + gamma(16) * raw_hi
        else:
            c = F.conv2d(xm, W, padding=layer.padding)
            ec = F.conv2d(x_abs, Wb, padding=layer.padding)
            if e_in is not None:
                ec = ec + F.conv2d(e_in, W.abs(), padding=layer.padding)
            c_hi = c.abs() + ec
            ec = ec + (H16 * c_hi + SUB16 * 2.0 ** e if fp16 else U32 * c_hi)
        del x_abs, e_in
        nz = (layer.noise_const.double() * layer.noise_strength.double()) if layer.use_noise else torch.zeros_like(c[0, 0])
        b = layer.bias.double()
        gain = layer.act_gain * kw.get('gain', 1)
        y, ey = tail_bound(c, ec, d, ed, nz, b, gain)

        def modulated(st, est, y=y, ey=ey):
            return y * _cv(st), ey * _cv(st.abs() + est) + y.abs() * _cv(est) + U32 * (y.abs() + ey) * _cv(st.abs() + est)

        block_next = self.chain_next.get(block)
        for kind, o in zip(kinds, outs):
            o = o[self.samples]
            if kind == 'y':
                ref, bound = y, ey
            elif kind == 'y*ys':
                ref, bound = modulated(*self.styles(block_next.conv0))
                assert bool(((cap['y_styles'].double() - self.styles(block_next.conv0)[0]).abs() <= self.styles(block_next.conv0)[1]).all())
            elif kind == 'y*sn':
                nxt = block.conv1 if layer is getattr(block, 'conv0', None) else block.torgb
                sn, esn = self.styles(nxt)
                assert bool(((cap['next_styles'].double() - sn).abs() <= esn).all()), f'{name}: next styles'
                ref, bound = modulated(sn, esn)
            else:
                wr, sr, br = cap['rgb']
                s_rgb, es_rgb = self.styles(block.torgb)
                assert wr is block.torgb.weight and br is block.torgb.bias
                Wr = wr.double().contiguous()
                ref = F.conv2d(y * _cv(s_rgb), Wr) + br.double()[None, :, None, None]
                t_hi = (y.abs() + ey) * _cv(s_rgb.abs() + es_rgb)
                bound = (F.conv2d(ey * _cv(s_rgb.abs() + es_rgb) + y.abs() * _cv(es_rgb), Wr.abs())
                         + gamma(Wr.shape[1] + 3) * (F.conv2d(t_hi, Wr.abs()) + br.double().abs()[None, :, None, None]))
                self.block_rgb[block] = (o.clone(), False)
            if o.dtype == torch.float16:
                bound = bound + H16 * (ref.abs() + bound) + SUB16
            self._record(name, kind, o, ref, bound)
            self._layer_controls(name, kind, o, ref, bound, c, d, nz, b, gain, modulated)
            del ref, bound
        self._end()

    def _layer_controls(self, name, kind, o, ref, bound, c, d, nz, b, gain, modulated):
        if kind == 'y*sn' and name in (self.controls.get('noise'), self.controls.get('bias'), self.controls.get('styles')):
            nxt_layer = self._next_of(name)
            sn, esn = self.styles(nxt_layer)
            y_shift = tail(c, d, torch.roll(nz, 1, dims=-1), b, gain)
            self._control('noise', name, o, ref, y_shift * _cv(sn), bound)
            b0 = b.clone()
            b0[4:8] = 0
            self._control('bias', name, o, ref, tail(c, d, nz, b0, gain) * _cv(sn), bound)
            self._control('styles', name, o, ref, tail(c, d, nz, b, gain) * _cv(sn.flip(0)), bound)
        if name == self.controls.get('tile'):
            # the last row of the 16 x 16 tile at tile row 1, tile column 2, channel block 1 (64 channels), where the shape has them
            C, H, Wd = o.shape[1:]
            r = min(31, H - 1)
            ch = slice(64, 128) if C >= 128 else slice(0, 64)
            cols = slice(32, 48) if Wd >= 48 else slice(0, 16)
            bad = ref.clone()
            bad[:, ch, r, cols] = ref[:, ch, r, cols] - o[:, ch, r, cols].double()      # the output row reads 0
            self._control('tile', name, o, ref, bad, bound)

    def _next_of(self, name):
        layer = dict(self.syn.named_modules())[name]
        block = self.block_of[layer]
        return block.conv1 if layer is getattr(block, 'conv0', None) else block.torgb

    def check_torgb(self, layer, cap, out):
        self._begin()
        name = self.names[layer]
        self.events.append((name, 'raw' if cap['raw'] else 'bias'))
        assert cap['premodulated'], f'{name}: ToRGB on a premodulated x'
        x = cap['x']
        o = out[self.samples]
        fp16 = x.dtype == torch.float16
        W = layer.weight.double().contiguous()
        mode = self._conv_mode(x, fp16)
        xm = x.double()
        ref = F.conv2d(xm, W)
        bound = F.conv2d(xm.abs(), conv_weight_bound(W, W.shape[1], mode))
        if fp16:                                   # an fp16 convolution writes fp16, also where the bias then comes on in float32
            bound = bound + H16 * (ref.abs() + bound) + SUB16
        else:
            bound = bound + U32 * (ref.abs() + bound)
        if not cap['raw']:
            b = layer.bias.double()[None, :, None, None]
            ref = ref + b
            bound = bound + U32 * (ref.abs() + bound + b.abs())
        self.calls.append(dict(stage=name, x=x.dtype, outs=(o.dtype,), fp16=fp16))
        self._record(name, 'torgb', o, ref, bound)
        self.block_rgb[self.block_of[layer]] = (o.clone(), cap['raw'])
        self._end()

    def check_skip(self, block, parts):
        """img_out = upsample2d(img_in) + y (+ b when the ToRGB output came raw), y the ToRGB / folded RGB output of this block."""
        self._begin()
        name = self.names[block]
        self.events.append((name, 'skip'))
        y, raw = self.block_rgb.pop(block)
        f = block.resample_filter.double()
        for img, out, sl in parts:
            o = out[self.samples]
            yy = y[:, sl].double()
            b = block.torgb.bias.double()[sl][None, :, None, None] if raw else torch.zeros_like(yy[:1, :, :1, :1])
            if img is None:
                up = up_abs = torch.zeros_like(yy)
            else:
                assert img.shape[-1] * 2 == yy.shape[-1]
                up, up_abs = oops.upsample2d(img.double(), f), oops.upsample2d(img.double().abs(), f)
            ref = up + yy + b
            bound = gamma(8) * (up_abs + yy.abs() + b.abs())
            assert o.dtype == torch.float32
            self._record(name, 'skip', o, ref, bound)
            if name == self.controls.get('skip') and img is not None:
                bad = ref.clone()
                bad[..., -1, :] = (yy + b)[..., -1, :]
                self._control('skip', name, o, ref, bad, bound)
            del ref, bound, up, up_abs
        self._end()

    def summary(self):
        """{stage kind: (largest err / bound, largest fp16 max|v| / 65504 | None)} -- the kind is the layer's role."""
        out = {}
        for ln in self.lines:
            role = ln['stage'].rsplit('.', 1)[-1] if '.' in ln['stage'] else 'skip'
            key = f"{'backbone' if ln['stage'].startswith('vb') else 'sr'} {role} {ln['kind']}"
            r, h = out.get(key, (0.0, None))
            hh = ln['headroom'] if h is None else (h if ln['headroom'] is None else max(h, ln['headroom']))
            out[key] = (max(r, ln['ratio']), hh)
        return out


def expected_events(synthesis, folded):
    """The call sequence of one synthesis call.  folded (NHWC chained path): the backbone's conv1 returns (y * s_next-block, y * s_rgb)
    (vb{last}: y * s_rgb alone), its ToRGB runs raw (but for the first block's), and the SR blocks fold ToRGB into conv1 ((y * s_next-block, rgb), then rgb alone).
    Unfolded (CPU oracle, NCHW): conv1 returns (y, y * s_rgb) and ToRGB adds its bias."""
    ev = []
    for chain, blocks in blocks_of(synthesis):
        for i, b in enumerate(blocks):
            n = [k for k, v in synthesis.named_modules() if v is b][0]
            last = i + 1 == len(blocks)
            ev.append((n, 'enter'))
            if b.in_channels:
                ev.append((f'{n}.conv0', ('y*sn',)))
            if not folded:
                ev += [(f'{n}.conv1', ('y', 'y*sn')), (f'{n}.torgb', 'bias')]
            elif chain == 'backbone':           # the first block has no running image to fuse the bias into: its ToRGB adds it
                ev += [(f'{n}.conv1', ('y*sn',) if last else ('y*ys', 'y*sn')), (f'{n}.torgb', 'raw' if i else 'bias')]
            else:
                ev.append((f'{n}.conv1', ('rgb',) if last else ('y*ys', 'rgb')))
            ev.append((n, 'skip'))
    return ev


DEFECTS = ('noise', 'bias', 'styles', 'tile', 'skip')


def run_checked(G, ws, c, monkeypatch, samples, controls, num_steps, **kw):
    chk = LayerChecker(G, ws, samples, controls)
    with monkeypatch.context() as mp:
        chk.install(mp)
        with torch.no_grad():
            G.synthesis(ws, c=c, render_params=dict(num_steps=num_steps), noise_mode='const', **kw)
    return chk


# ------------------------------------------------------------------------------------------------ GPU: the benchmark's generator
@pytest.fixture(scope='module')
def bench_case():
    from bench import NUM_STEPS, make_labels, make_latents
    from ide3d_b200.compat import random_init_generator
    G = switch_on_terms(random_init_generator(device='cuda', seed=0))
    with torch.no_grad():
        ws = G.mapping(make_latents(8, G.z_dim).cuda(), make_labels(8).cuda())
    yield G, ws, make_labels(8).cuda(), NUM_STEPS
    del G
    torch.cuda.empty_cache()


GPU_CONTROLS = dict(noise='vb64.conv1', bias='vb64.conv1', styles='vb64.conv1', tile='vb64.conv0', skip='vb128')


@pytest.mark.gpu
@pytest.mark.parametrize('tf32', [False, True])
def test_bench_synthesis_layers_against_float64(bench_case, monkeypatch, tf32):
    from ide3d_b200.training import networks
    G, ws, c, steps = bench_case
    syn = G.synthesis
    backbone = blocks_of(syn)[0][1]
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cudnn.benchmark)
    t0 = time.perf_counter()
    try:
        torch.backends.cudnn.allow_tf32, torch.backends.cudnn.benchmark = tf32, True
        assert networks.fp16_operands(backbone) == tf32
        with torch.no_grad():
            assert syn._style_plan(ws) is not None
        assert all(b.torgb.weight.shape[0] <= 4 and b.can_fold() for b in blocks_of(syn)[1][1])      # both SR blocks fold ToRGB
        chk = run_checked(G, ws, c, monkeypatch, [0, ws.shape[0] - 1], GPU_CONTROLS, steps, perturb='hash', seed=7)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cudnn.benchmark = prev
    props = torch.cuda.get_device_properties(0)
    print(f'{props.name}, tf32={tf32}: negative controls, max err/bound', {k: round(v, 1) for k, v in chk.rejected.items()})
    print(f'{props.name}, tf32={tf32}: {len(chk.lines)} outputs checked in {time.perf_counter() - t0:.1f} s, float64 peak '
          f'{chk.peak / 2 ** 30:.2f} GiB')
    for k, (r, h) in chk.summary().items():
        print(f'  {k:<28s} max err/bound {r:.3f}' + ('' if h is None else f'  fp16 max|v|/65504 {h:.2e}'))
    assert chk.events == expected_events(syn, folded=True)
    assert len(syn.voxel_block_resolutions) == 7 and len(syn.block_resolutions) == 2
    # the path that ran, from the dtypes: fp16 operands in the backbone exactly under TF32, float32 everywhere in the SR blocks
    for call in chk.calls:
        half = tf32 and call['stage'].startswith('vb')
        want = torch.float16 if half else torch.float32
        out = torch.float32 if call['stage'] == 'vb4.torgb' else want                                 # ToRGB with its bias: float32
        assert call['fp16'] == half and all(o == out for o in call['outs']), call
        assert call['x'] == (torch.float32 if call['stage'] == 'vb4.conv1' else want), call          # vb4's constant comes in float32
    assert sorted(chk.rejected) == sorted(DEFECTS) and all(r > 1 for r in chk.rejected.values()), chk.rejected


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1, 8, 11])
def test_bench_style_plan_against_float64(bench_case, n):
    """StylePlan at the bench generator: 26 entries (20 backbone, 6 SR), w_dim 512.  style_plan.cu walks the batch in passes of
    kStyleBatch = 8 samples, so n = 11 takes a ragged second pass.  Styles and dcoefs within their float32 bounds of the float64 values;
    fp16_blocks multiplies the backbone's dcoefs by exactly 2^e (bit for bit) and leaves everything else as it was."""
    from bench import make_labels, make_latents
    from ide3d_b200.training import triplane
    G = bench_case[0]
    syn = G.synthesis
    backbone = blocks_of(syn)[0][1]
    with torch.no_grad():
        ws = G.mapping(make_latents(n, G.z_dim, offset=100).cuda(), make_labels(n).cuda())
        plan = syn._style_plan(ws)
        plan16 = syn._style_plan(ws, fp16_blocks=backbone)
    sp = triplane._STYLE_PLANS[syn]
    assert len(sp.entries) == 26 and syn.w_dim == 512
    bb = {m for b in backbone for m in b.modules()}
    assert sum(layer in bb for layer, *_ in sp.entries) == 20
    rows = ws_rows(syn)
    for layer, (s, d) in plan.items():
        s_ref, es = style_ref(layer, ws[:, rows[layer]])
        assert bool(((s.double() - s_ref).abs() <= es).all()), (layer, float(((s.double() - s_ref).abs() / es).max()))
        s16, d16 = plan16[layer]
        assert torch.equal(s16, s)
        if d is None:
            assert d16 is None
            continue
        d_ref, ed = demod_ref(layer, s_ref, es)
        assert bool(((d.double() - d_ref).abs() <= ed).all()), (layer, float(((d.double() - d_ref).abs() / ed).max()))
        e = layer.fp16_exponent() if layer in bb else 0
        assert torch.equal(d16, d * 2.0 ** e), layer


# ------------------------------------------------------------------------------------------------ CPU rehearsal
def test_layer_checker_rehearsal_on_cpu(monkeypatch):
    """The checker above on a reduced generator under the CPU oracle: NCHW, no style plan, unfolded ToRGB with its bias, _accumulate.
    Every call is checked, the sequence holds and every negative control is rejected."""
    from oracle.backend import cpu_reference_ops
    from ide3d_b200.training.triplane import TriPlaneGenerator
    torch.manual_seed(0)
    G = TriPlaneGenerator(z_dim=16, w_dim=16, img_resolution=32, plane_resolution=32, render_size=8, channel_base=512,
                          channel_max=128, sr_channels=(16, 8), mapping_kwargs=dict(num_layers=1)).eval().requires_grad_(False)
    switch_on_terms(G)
    n = 3
    g = torch.Generator().manual_seed(2)
    c = torch.tensor([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1.]).repeat(n, 1)
    controls = dict(noise='vb16.conv1', bias='vb16.conv1', styles='vb16.conv1', tile='vb32.conv0', skip='vb32')
    with cpu_reference_ops():
        with torch.no_grad():
            ws = G.mapping(torch.randn(n, 16, generator=g), c)
        chk = run_checked(G, ws, c, monkeypatch, [0, n - 1], controls, 6, perturb=None)
    syn = G.synthesis
    assert chk.events == expected_events(syn, folded=False)
    blocks = [b for _, bl in blocks_of(syn) for b in bl]
    assert len(chk.calls) == sum(3 if b.in_channels else 2 for b in blocks)         # every layer and every ToRGB call
    # outputs: conv0 y * s1, conv1 (y, y * s_rgb), ToRGB, and one skip image per output (two in the dual-path backbone blocks)
    assert len(chk.lines) == sum(int(b.in_channels != 0) + 2 + 1 + (2 if b in blocks_of(syn)[0][1] else 1) for b in blocks)
    assert all(call['x'] == torch.float32 and not call['fp16'] for call in chk.calls)
    assert sorted(chk.rejected) == sorted(DEFECTS) and all(r > 1 for r in chk.rejected.values()), chk.rejected
