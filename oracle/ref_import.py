"""ORACLE / TEST INFRASTRUCTURE ONLY — never imported by the product path.

Imports the reference's own modules VERBATIM from a checkout of autonomousvision/transfuser (branch 2022) — the directory
named by $TRANSFUSER_REFERENCE, by default `reference/` next to this repository — behind the shim packages in oracle/shims for the
un-vendored dependencies (timm, mmcv, mmdet, torch_scatter).  Used to (1) validate the CPU
restatement in oracle/torch_oracle.py and (2) generate the committed fixtures in tests/golden/
(oracle/make_golden.py).
"""
import importlib
import os
import sys

REF_ROOT = os.path.join(os.environ.get('TRANSFUSER_REFERENCE', os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), 'reference')),
                        'team_code_transfuser')
SHIMS = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'shims')


def available():
    return os.path.isfile(os.path.join(REF_ROOT, 'transfuser.py'))


def load():
    """Returns the reference modules (config, transfuser, model) imported unmodified."""
    if not available():
        raise RuntimeError('reference not present at %s' % REF_ROOT)
    for p in (SHIMS, REF_ROOT):
        if p not in sys.path:
            sys.path.insert(0, p)
    mods = {}
    for name in ('config', 'transfuser', 'model'):
        mods[name] = importlib.import_module(name)
    return mods


def load_histogram_fn():
    """`lidar_to_histogram_features` (data.py:446-470) exec'd alone: data.py itself needs ujson/skimage."""
    import numpy as np
    src = open(os.path.join(REF_ROOT, 'data.py')).read().split('\n')
    start = next(i for i, l in enumerate(src) if l.startswith('def lidar_to_histogram_features'))
    end = next(i for i in range(start + 1, len(src)) if src[i].startswith('def '))
    ns = {'np': np}
    exec('\n'.join(src[start:end]), ns)
    return ns['lidar_to_histogram_features']


def load_data_fns(names):
    """Functions of data.py exec'd one by one from the file's own text (data.py as a module needs ujson / skimage, which are
    not in the image): the reference's utils.py is imported verbatim for the transforms, cv2 is the real OpenCV, and `np` is
    numpy plus the `np.float` alias that data.py:630 still uses (removed in numpy 1.24)."""
    import ast
    import types
    import cv2
    import numpy as np
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    utils = importlib.import_module('utils')
    npx = types.ModuleType('np_with_float_alias')
    npx.__dict__.update(np.__dict__)
    npx.float = float
    text = open(os.path.join(REF_ROOT, 'data.py')).read()
    ns = {'np': npx, 'cv2': cv2}
    ns.update({k: getattr(utils, k) for k in dir(utils) if k.startswith('get_')})
    wanted = set(names)
    for node in ast.parse(text).body:
        if isinstance(node, ast.FunctionDef) and node.name in wanted:
            exec(compile(ast.Module(body=[node], type_ignores=[]), os.path.join(REF_ROOT, 'data.py'), 'exec'), ns)
    missing = wanted - set(ns)
    if missing:
        raise RuntimeError('not found in data.py: %s' % sorted(missing))
    return {k: ns[k] for k in names}
