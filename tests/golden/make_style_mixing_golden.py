"""Golden data of the style-mixing rule: the reference's own lines, loaded from its source and run on the CPU.

    python tests/golden/make_style_mixing_golden.py [/path/to/reference]   -> tests/golden/style_mixing.npz

From apps/style_mixing.py: num_range; the w draw, mapping and truncation (:90-95); the mixing of each cell (:113-114); the key
choice of the canvas loop (:141-150), which gives the canvas order.  From viz/renderer.py: the filter of the style rows (:331).
They run with oracle.style_mixing.StandInMapping (seed 0) as G2.generator.mapping, and the mapping's label argument (None in the
reference) replaced by the frontal camera label, the deviation ide3d_b200.style_mixing documents.  Stored per case: the inputs and
the ws of every cell in canvas order [(R+1)(C+1) - 1, 18, 8]."""

import ast
import contextlib
import io
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

FRONTAL = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 2.7, 0, 0, 0, 1, 4.2647, 0, 0.5, 0, 4.2647, 0.5, 0, 0, 1]
CASES = {                                   # rows, cols, styles (a --styles string), psi
    'overlap': ('1,2,3', '2,5', '0-6', 1.0),
    'single_row': ('4', '7,8,9', '14-17', 0.7),
    'single_col': ('3,11,12', '6', '8,9,10', 1.0),
    'out_of_range': ('1,2', '3,1', '16,17,18,25', 1.0),
    'psi': ('0,1', '1,2,3', '0-17', 0.5),
}
NUM_RANGE = ('0-6', '14-17', '3,5,9', '7', '10-10')


def _function(tree, name):
    return next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == name)


def reference_pieces(ref):
    """(num_range, w-draw source, cell-mix source, canvas-key source, style-filter source) from the reference tree."""
    tree = ast.parse(open(os.path.join(ref, 'apps', 'style_mixing.py')).read())
    ns = {'re': __import__('re'), 'List': list}
    exec(compile(ast.Module(body=[_function(tree, 'num_range')], type_ignores=[]), 'style_mixing.py', 'exec'), ns)
    body = _function(tree, 'generate_style_mix').body
    src = [ast.unparse(s) for s in body]
    draw = [s for s in src if s.split(' = ')[0] in ('all_seeds', 'all_z', 'all_w', 'w_avg', 'w_dict')]
    assert len(draw) == 6, draw
    draw = [s.replace(', None)', ', c_label)') for s in draw]           # the frontal label instead of c=None
    mix_loop = next(s for s in body if isinstance(s, ast.For) and ast.unparse(s.target) == 'row_seed')
    inner = mix_loop.body[0]
    mix = [ast.unparse(s) for s in inner.body[:2]]
    assert mix[0].startswith('w = w_dict[row_seed].clone()') and mix[1].startswith('w[col_styles]'), mix
    step_loop = next(s for s in body if isinstance(s, ast.For) and ast.unparse(s.target) == 'step')
    canvas_loop = step_loop.body[1]
    assert ast.unparse(canvas_loop.target).strip('()') == 'row_idx, row_seed', ast.unparse(canvas_loop)
    col_loop = canvas_loop.body[0]
    keys = [ast.unparse(s) for s in col_loop.body[:4]]
    assert keys[1].startswith('key = (row_seed, col_seed)'), keys
    viz = ast.parse(open(os.path.join(ref, 'viz', 'renderer.py')).read())
    filt = [ast.unparse(n) for n in ast.walk(viz) if isinstance(n, ast.Assign) and ast.unparse(n.targets[0]) == 'stylemix_idx'
            and 'num_ws' in ast.unparse(n.value)]
    assert len(filt) == 1, filt
    return ns['num_range'], draw, mix, keys, filt[0]


def run_case(pieces, G, rows, cols, styles, psi):
    num_range, draw, mix, keys, filt = pieces
    with contextlib.redirect_stdout(io.StringIO()):                     # num_range prints its argument
        row_seeds, col_seeds, col_styles = num_range(rows), num_range(cols), num_range(styles)
    ns = dict(np=np, torch=torch, G=G, G2=types.SimpleNamespace(generator=G), device='cpu', truncation_psi=psi,
              row_seeds=row_seeds, col_seeds=col_seeds, c_label=None)
    # viz/renderer.py:331 on the style rows, with G.backbone.num_ws the generator's num_ws
    ns_f = dict(stylemix_idx=col_styles, G=types.SimpleNamespace(backbone=types.SimpleNamespace(num_ws=G.num_ws)))
    exec(filt, ns_f)
    ns['col_styles'] = ns_f['stylemix_idx']
    all_seeds_n = len(set(row_seeds + col_seeds))
    ns['c_label'] = torch.tensor(FRONTAL).float().reshape(1, -1).repeat(all_seeds_n, 1)
    for s in draw:
        exec(s, ns)
    mixed = {}
    for row_seed in row_seeds:
        for col_seed in col_seeds:
            ns.update(row_seed=row_seed, col_seed=col_seed)
            for s in mix:
                exec(s, ns)
            mixed[(row_seed, col_seed)] = ns['w']
    cell_ws = {(s, s): w for s, w in ns['w_dict'].items()}
    cell_ws.update(mixed)
    order = []
    for row_idx, row_seed in enumerate([0] + row_seeds):
        for col_idx, col_seed in enumerate([0] + col_seeds):
            k = dict(row_idx=row_idx, row_seed=row_seed, col_idx=col_idx, col_seed=col_seed)
            if row_idx == 0 and col_idx == 0:
                continue
            exec('\n'.join(keys[1:]), k)
            order.append(k['key'])
    return row_seeds, col_seeds, ns['col_styles'], order, torch.stack([cell_ws[key] for key in order]).numpy()


def main(ref=None):
    ref = ref or os.environ.get('IDE3D_REFERENCE', '/root/reference')
    from oracle.style_mixing import stand_in_generator
    pieces = reference_pieces(ref)
    G = stand_in_generator(seed=0)
    out = {}
    with contextlib.redirect_stdout(io.StringIO()):
        for s in NUM_RANGE:
            out[f'num_range/{s}'] = np.array(pieces[0](s), dtype=np.int64)
    for name, (rows, cols, styles, psi) in CASES.items():
        r, c, st, order, ws = run_case(pieces, G, rows, cols, styles, psi)
        out[f'{name}/rows'], out[f'{name}/cols'] = np.array(r, np.int64), np.array(c, np.int64)
        out[f'{name}/styles_arg'], out[f'{name}/styles_kept'] = np.array(styles), np.array(st, np.int64)
        out[f'{name}/psi'], out[f'{name}/order'], out[f'{name}/ws'] = np.float64(psi), np.array(order, np.int64), ws
    path = os.path.join(HERE, 'style_mixing.npz')
    np.savez_compressed(path, **out)
    print(path, {k: v.shape for k, v in out.items() if k.endswith('/ws')})


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else None)
