"""ModelConfig.loss without a GPU: losses.resolve in every accepted form and every refusal, the float64 restatement
(tests/loss_ref.py) at the edges where TensorFlow's gradient conventions decide, and pickling."""
import math
import pickle

import numpy as np
import pytest
import torch

import loss_ref
from deeptables_b200 import losses as LS

KINDS = list(LS._CLASSES)
FUNCTIONS = {'MeanSquaredError': 'mean_squared_error', 'MeanAbsoluteError': 'mean_absolute_error',
             'MeanAbsolutePercentageError': 'mean_absolute_percentage_error',
             'MeanSquaredLogarithmicError': 'mean_squared_logarithmic_error', 'Huber': 'huber', 'LogCosh': 'log_cosh',
             'Poisson': 'poisson', 'Hinge': 'hinge', 'SquaredHinge': 'squared_hinge',
             'CategoricalHinge': 'categorical_hinge', 'KLDivergence': 'kl_divergence',
             'BinaryCrossentropy': 'binary_crossentropy', 'CategoricalCrossentropy': 'categorical_crossentropy'}
ALIASES = {'mse': 'MeanSquaredError', 'mae': 'MeanAbsoluteError', 'mape': 'MeanAbsolutePercentageError',
           'msle': 'MeanSquaredLogarithmicError', 'kld': 'KLDivergence', 'bce': 'BinaryCrossentropy'}


def _keras_like(class_name, config):
    """An object shaped like a real keras.losses instance: its class name and get_config()."""
    return type(class_name, (), {'get_config': lambda self: dict(config)})()


def _keras_function(name):
    def fn(y_true, y_pred):
        raise AssertionError('never called')
    fn.__name__ = name
    fn.__module__ = 'keras.src.losses.losses'
    return fn


# ---- resolve: accepted forms ------------------------------------------------------------------------------------------
def test_the_codes_follow_the_header():
    import re
    from deeptables_b200 import _native
    with open(_native.HEADER_PATH) as f:
        header = dict((m[0], int(m[1])) for m in re.findall(r'#define DTB_LOSS_([A-Z_]+) (\d+)', f.read()))
    assert len(header) == len(KINDS) == 13
    for kind, code in LS.CODES.items():
        assert header[re.sub(r'(?<!^)(?=[A-Z])', '_', kind).upper().replace('K_L_', 'KL_')] == code, kind


@pytest.mark.parametrize('kind', KINDS)
def test_every_form_resolves_to_the_same_spec(kind):
    want = LS.LossSpec(kind)
    cls = getattr(LS, kind)
    keras_config = {'name': FUNCTIONS[kind], 'reduction': 'sum_over_batch_size',
                    'dtype': {'module': 'keras', 'class_name': 'DTypePolicy', 'config': {'name': 'float32'}}}
    if kind == 'Huber':
        keras_config['delta'] = 1.0
    if 'Crossentropy' in kind:
        keras_config.update(from_logits=False, label_smoothing=0.0, axis=-1)
    forms = [cls(), kind, kind.lower(), kind.upper(), FUNCTIONS[kind], FUNCTIONS[kind].upper(),
             _keras_like(kind, keras_config), {'class_name': kind, 'config': keras_config}, {'class_name': kind},
             _keras_function(FUNCTIONS[kind]), {'class_name': 'function', 'config': FUNCTIONS[kind]}, want]
    forms += [alias for alias, k in ALIASES.items() if k == kind]
    for form in forms:
        assert LS.resolve(form, 'binary') == want, repr(form)


def test_parameters_are_read_from_every_form():
    assert LS.resolve(LS.Huber(delta=2.5), 'regression') == LS.LossSpec('Huber', 2.5, 0.0)
    assert LS.resolve(LS.Huber(0.25), 'regression').delta == 0.25                     # positional, as Keras
    assert LS.resolve(_keras_like('Huber', {'delta': 3, 'name': 'h'}), 'regression').delta == 3.0
    assert LS.resolve({'class_name': 'Huber', 'config': {'delta': 0.5}}, 'regression').delta == 0.5
    for cls in (LS.BinaryCrossentropy, LS.CategoricalCrossentropy):
        spec = LS.resolve(cls(label_smoothing=0.1), 'binary')
        assert spec == LS.LossSpec(cls.__name__, 1.0, 0.1)
        assert LS.resolve(_keras_like(cls.__name__, {'label_smoothing': 1, 'from_logits': False}), 'binary') \
            .label_smoothing == 1.0
    assert LS.resolve(LS.MeanSquaredError(reduction='sum_over_batch_size', name='m', dtype='float32'), 'binary') == \
        LS.LossSpec('MeanSquaredError')


def test_names_and_builtin_pairs():
    assert str(LS.resolve('mse', 'regression')) == 'mean_squared_error'
    assert str(LS.resolve(LS.Huber(delta=2.0), 'regression')) == 'huber(delta=2.0)'
    assert str(LS.resolve(LS.Huber(), 'regression')) == 'huber'
    assert str(LS.resolve(LS.BinaryCrossentropy(label_smoothing=0.1), 'binary')) == \
        'binary_crossentropy(label_smoothing=0.1)'
    builtin = {('BinaryCrossentropy', 'binary'), ('BinaryCrossentropy', 'multilabel'), ('MeanSquaredError', 'regression'),
               ('CategoricalCrossentropy', 'multiclass')}
    for kind in KINDS:
        for task in ('binary', 'multilabel', 'regression', 'multiclass'):
            assert LS.LossSpec(kind).builtin(task) == ((kind, task) in builtin), (kind, task)
    assert not LS.LossSpec('BinaryCrossentropy', label_smoothing=0.1).builtin('binary')
    assert not LS.LossSpec('CategoricalCrossentropy', label_smoothing=0.1).builtin('multiclass')
    assert LS.LossSpec('Hinge').hinge and LS.LossSpec('SquaredHinge').hinge and not LS.LossSpec('CategoricalHinge').hinge


# ---- resolve: refusals ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('loss,option', [
    (LS.BinaryCrossentropy(from_logits=True), 'from_logits'),
    (LS.CategoricalCrossentropy(from_logits=True), 'from_logits'),
    (LS.MeanSquaredError(reduction='sum'), 'reduction'),
    (LS.Huber(reduction=None), 'reduction'),
    ({'class_name': 'MeanAbsoluteError', 'config': {'reduction': 'mean_with_sample_weight'}}, 'reduction'),
    (LS.CategoricalCrossentropy(axis=1), 'axis'),
    (LS.Poisson(dtype='float16'), 'dtype'),
    (_keras_like('Hinge', {'dtype': {'class_name': 'DTypePolicy', 'config': {'name': 'mixed_float16'}}}), 'dtype'),
    (_keras_like('Huber', {'delta': 1.0, 'fn': 'x'}), 'fn'),
    ('cosine_similarity', 'cosine_similarity'),
    ('CosineSimilarity', 'CosineSimilarity'),
    (_keras_like('CosineSimilarity', {'axis': -1}), 'CosineSimilarity'),
    (_keras_like('BinaryFocalCrossentropy', {}), 'BinaryFocalCrossentropy'),
    ({'class_name': 'CategoricalFocalCrossentropy', 'config': {}}, 'CategoricalFocalCrossentropy'),
    ('tversky', 'tversky'),
    (lambda y, p: (y - p) ** 2, 'custom loss functions'),
    (_keras_function('cosine_similarity'), 'custom loss functions'),
    (LS.Huber, 'not the class'),
    (None, 'None'),
    (3, '3'),
])
def test_options_that_are_not_built_raise_not_implemented(loss, option):
    with pytest.raises(NotImplementedError, match=option):
        LS.resolve(loss, 'binary')


@pytest.mark.parametrize('loss', [
    'sparse_categorical_crossentropy', 'SparseCategoricalCrossentropy', _keras_like('SparseCategoricalCrossentropy', {}),
    {'class_name': 'SparseCategoricalCrossentropy', 'config': {}}, _keras_function('sparse_categorical_crossentropy')])
def test_sparse_categorical_crossentropy_is_a_value_error(loss):
    with pytest.raises(ValueError, match='one-hot'):
        LS.resolve(loss, 'multiclass', 4)


@pytest.mark.parametrize('loss', [
    LS.BinaryCrossentropy(label_smoothing=-0.1), LS.CategoricalCrossentropy(label_smoothing=1.5),
    LS.BinaryCrossentropy(label_smoothing=float('nan')), LS.BinaryCrossentropy(label_smoothing=True),
    LS.Huber(delta=0.0), LS.Huber(delta=-1.0), LS.Huber(delta=float('inf')), LS.Huber(delta=float('nan')),
    LS.Huber(delta='1')])
def test_bad_values_are_value_errors(loss):
    with pytest.raises(ValueError):
        LS.resolve(loss, 'binary')


def test_unknown_constructor_arguments_are_type_errors():
    with pytest.raises(TypeError):
        LS.Huber(delta=1.0, gamma=2.0)
    with pytest.raises(TypeError):
        LS.MeanSquaredError('sum_over_batch_size', 'n', None, 4)


# ---- pickling ---------------------------------------------------------------------------------------------------------------
def test_losses_and_configs_pickle():
    from deeptables_b200 import deeptable
    for loss in [getattr(LS, k)() for k in KINDS] + [LS.Huber(delta=2.0), LS.CategoricalCrossentropy(label_smoothing=0.2)]:
        back = pickle.loads(pickle.dumps(loss))
        assert type(back) is type(loss) and back.get_config() == loss.get_config()
        assert LS.resolve(back, 'binary') == LS.resolve(loss, 'binary')
    spec = LS.LossSpec('Huber', 2.0)
    assert pickle.loads(pickle.dumps(spec)) == spec and hash(spec) == hash(LS.LossSpec('Huber', 2.0))
    conf = deeptable.ModelConfig(loss=LS.Huber(delta=0.5))
    assert LS.resolve(pickle.loads(pickle.dumps(conf)).loss, 'regression') == LS.LossSpec('Huber', 0.5)


# ---- the float64 restatement at its edges -------------------------------------------------------------------------------
def _grad(kind, y, p, **kw):
    p = torch.tensor(p, dtype=torch.float64, requires_grad=True)
    y = torch.tensor(y, dtype=torch.float64)
    loss = loss_ref.per_row(kind, y, p, **kw)
    (g,) = torch.autograd.grad(loss.sum(), [p])
    return loss.detach().numpy(), g.numpy()


def test_huber_at_delta_is_quadratic():
    loss, g = _grad('Huber', [[0.25, 0.25]], [[0.75, -0.25]], delta=0.5)      # |e| = delta in both columns
    np.testing.assert_allclose(loss, [0.125], rtol=1e-15)
    np.testing.assert_allclose(g, [[0.25, -0.25]], rtol=1e-15)                 # e / C, the quadratic branch
    loss, g = _grad('Huber', [[0.0]], [[2.0]], delta=0.5)
    np.testing.assert_allclose(loss, [0.5 * 2.0 - 0.125])
    np.testing.assert_allclose(g, [[0.5]])


def test_hinge_at_the_margin_passes_the_label():
    # 0 / 1 labels become -1 / 1: y' p = 1 exactly, the gradient is -y' / C
    loss, g = _grad('Hinge', [[1.0, 0.0]], [[1.0, -1.0]])
    np.testing.assert_allclose(loss, [0.0])
    np.testing.assert_allclose(g, [[-0.5, 0.5]])
    loss, g = _grad('SquaredHinge', [[1.0, 0.0]], [[1.0, -1.0]])
    np.testing.assert_allclose(g, [[0.0, 0.0]])
    # a label outside {0, 1} anywhere in the batch: no conversion, y' = y
    loss, g = _grad('Hinge', [[1.0, 0.0], [0.5, 0.0]], [[0.2, 0.3], [0.0, 0.0]])
    np.testing.assert_allclose(loss, [(0.8 + 1.0) / 2, 1.0])
    np.testing.assert_allclose(g, [[-0.5, 0.0], [-0.25, 0.0]])


def test_mape_at_a_zero_label_divides_by_epsilon():
    loss, g = _grad('MeanAbsolutePercentageError', [[0.0, 2.0]], [[0.5, 1.0]])
    np.testing.assert_allclose(loss, [100.0 * (0.5 / loss_ref.EPS + 0.5) / 2], rtol=1e-12)
    np.testing.assert_allclose(g, [[100.0 / loss_ref.EPS / 2, -100.0 / 2.0 / 2]], rtol=1e-12)


def test_below_epsilon_msle_and_kl_take_no_gradient():
    loss, g = _grad('MeanSquaredLogarithmicError', [[1.0, 1.0]], [[-0.5, 1e-8]])
    want = (math.log(1 + loss_ref.EPS) - math.log(2.0)) ** 2
    np.testing.assert_allclose(loss, [want], rtol=1e-12)
    np.testing.assert_array_equal(g, [[0.0, 0.0]])
    loss, g = _grad('KLDivergence', [[0.5, 0.5]], [[1e-9, 1.5]])
    np.testing.assert_allclose(loss, [0.5 * math.log(0.5 / loss_ref.EPS) + 0.5 * math.log(0.5)], rtol=1e-12)
    np.testing.assert_array_equal(g, [[0.0, 0.0]])


def test_categorical_hinge_splits_tied_maxima():
    # (1 - y) p = [0.3, 0.3, 0]: two tied maxima share the gradient of neg
    loss, g = _grad('CategoricalHinge', [[0.0, 0.0, 1.0]], [[0.3, 0.3, 0.4]])
    np.testing.assert_allclose(loss, [0.3 - 0.4 + 1.0], rtol=1e-12)
    np.testing.assert_allclose(g, [[0.5, 0.5, -1.0]], rtol=1e-15)


def test_label_smoothing_moves_the_targets():
    y, p = [[1.0, 0.0]], [[0.7, 0.2]]
    s = 0.2
    got, _ = _grad('BinaryCrossentropy', y, p, label_smoothing=s)
    ys = np.array([0.9, 0.1])
    want = -np.mean(ys * np.log(p[0]) + (1 - ys) * np.log(1 - np.array(p[0])))
    np.testing.assert_allclose(got, [want], rtol=1e-12)
    got, g = _grad('CategoricalCrossentropy', y, p, label_smoothing=s)
    q = np.array(p[0]) / 0.9
    ys = np.array([0.9, 0.1])
    np.testing.assert_allclose(got, [-(ys * np.log(q)).sum()], rtol=1e-12)
    # the renormalisation: scaling p leaves the loss unchanged, so the gradient is orthogonal to p
    assert abs(float((g * np.array(p)).sum())) < 1e-12
