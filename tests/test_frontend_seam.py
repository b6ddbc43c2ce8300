"""CPU checks of the seam between recognition and training at the front end: the front-end forward kernels are launched
only from modules.py, whose front-end classes hold the one forward both paths run (modules.encoder_input_bf16) and the
backward beside it; train.py neither reads an encoder's private rel-pos cache nor asks which front end it holds."""
import ast
import os
import re

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'opentransformer_b200')
FRONT_END_KERNELS = ('conv1_relu', 'conv2_relu', 'frame_stack')
FRONT_END_CLASSES = ('ConvFrontEnd', 'ConcatFeatureFrontEnd', 'ConcatWithLinearFrontEnd')


def _source(name):
    with open(os.path.join(PKG, name)) as f:
        return f.read()


def test_front_end_kernels_are_called_only_from_modules_py():
    bad = []
    for name in sorted(os.listdir(PKG)):
        if name.endswith('.py') and name not in ('modules.py', 'ops.py'):
            bad += [f'{name}: ops.{k}' for k in FRONT_END_KERNELS if re.search(rf'\bops\.{k}\(', _source(name))]
    assert not bad, 'front-end kernels outside modules.py:\n' + '\n'.join(bad)


def test_train_py_runs_the_shared_front_half():
    text = _source('train.py')
    assert '_rel_pos' not in text
    assert 'EPI_TABLE' not in text
    assert 'encoder_input_bf16' in text and 'frontend.backward(' in text


def test_train_py_does_not_dispatch_on_the_front_end_class():
    """No isinstance on a front-end class outside EncoderPack, whose constructor refuses what training does not cover."""
    tree = ast.parse(_source('train.py'))
    bad = []
    for top in tree.body:
        if isinstance(top, ast.ClassDef) and top.name == 'EncoderPack':
            scopes = [f for f in top.body if isinstance(f, ast.FunctionDef) and f.name != '__init__']
        else:
            scopes = [top]
        for scope in scopes:
            for node in ast.walk(scope):
                if isinstance(node, ast.Name) and node.id in FRONT_END_CLASSES:
                    bad.append(f'{getattr(scope, "name", type(scope).__name__)}: {node.id} (line {node.lineno})')
    assert not bad, 'train.py names a front-end class outside the EncoderPack checks:\n' + '\n'.join(bad)
