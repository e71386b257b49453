"""Keras weight regularizers without a GPU: what ``regularizers.resolve`` accepts and rejects, the regularized
parameters' segments of the flat parameter buffer, and the float64 formulas of reg_ref.py against torch.autograd."""
import math

import pytest
import torch

import reg_ref
from deeptables_b200 import regularizers as R


class L2:
    """Stand-in for keras.regularizers.L2: only the class name and get_config() count."""

    def __init__(self, l2):
        self.l2 = l2

    def get_config(self):
        return {'l2': self.l2}


class OrthogonalRegularizer:
    def get_config(self):
        return {'factor': 0.01, 'mode': 'rows'}


@pytest.mark.parametrize('arg,want', [
    (None, None),
    ('l1', (0.01, 0.0)), ('L1', (0.01, 0.0)),
    ('l2', (0.0, 0.01)), ('L2', (0.0, 0.01)),
    ('l1_l2', None), ('L1L2', None),                       # Keras's L1L2() defaults to 0, 0
    (R.L1(), (0.01, 0.0)), (R.L1(0.5), (0.5, 0.0)), (R.L1(l1=None), (0.01, 0.0)),
    (R.L2(), (0.0, 0.01)), (R.L2(l2=3e-5), (0.0, 3e-5)),
    (R.L1L2(), None), (R.L1L2(0.0, 0.0), None), (R.L1L2(l1=1e-3), (1e-3, 0.0)), (R.L1L2(1e-3, 2e-3), (1e-3, 2e-3)),
    ({'class_name': 'L2', 'config': {'l2': 1e-5}}, (0.0, 1e-5)),
    ({'module': 'keras.regularizers', 'class_name': 'L1L2', 'config': {'l1': 0.1, 'l2': 0.2},
      'registered_name': None}, (0.1, 0.2)),
    ({'class_name': 'L1', 'config': {}}, (0.01, 0.0)),
    (L2(0.25), (0.0, 0.25)),
    (R.RegSpec(0.1, 0.0), (0.1, 0.0)),
])
def test_resolve_accepted_forms(arg, want):
    spec = R.resolve(arg)
    if want is None:
        assert spec is None
    else:
        assert isinstance(spec, R.RegSpec) and tuple(spec) == want


def test_get_config_round_trips():
    for reg in (R.L1(0.2), R.L2(0.3), R.L1L2(0.1, 0.4)):
        cfg = reg.get_config()
        again = type(reg)(**cfg)
        assert again.get_config() == cfg
        assert R.resolve({'class_name': type(reg).__name__, 'config': cfg}) == R.resolve(reg)
    assert R.L1L2().get_config() == {'l1': 0.0, 'l2': 0.0}


@pytest.mark.parametrize('make', [lambda: R.L1(-0.1), lambda: R.L2(-1e-9), lambda: R.L1L2(l1=-1.0),
                                  lambda: R.L2(float('nan')), lambda: R.L1(math.inf), lambda: R.L1L2(l2='0.1'),
                                  lambda: R.resolve({'class_name': 'L2', 'config': {'l2': -0.5}}),
                                  lambda: R.resolve(L2(-0.5))])
def test_negative_or_non_finite_factors_raise_value_error(make):
    with pytest.raises(ValueError):
        make()


@pytest.mark.parametrize('arg,needle', [
    (OrthogonalRegularizer(), 'OrthogonalRegularizer'),
    ('orthogonal_regularizer', 'OrthogonalRegularizer'),
    ({'class_name': 'OrthogonalRegularizer', 'config': {}}, 'OrthogonalRegularizer'),
    (lambda w: 0.01 * w.sum(), 'callable'),
    ('l3', 'not built natively'),
])
def test_unsupported_regularizers_raise(arg, needle):
    with pytest.raises(NotImplementedError, match=needle):
        R.resolve(arg)


def test_activity_regularizers_raise():
    from deeptables_b200 import layers
    with pytest.raises(NotImplementedError, match='activity'):
        layers.Dense(4, activity_regularizer=R.L2())
    with pytest.raises(NotImplementedError, match='activity'):
        R.reject_activity('l2', 'embeddings_activity_regularizer')
    R.reject_activity(None, 'embeddings_activity_regularizer')


def test_layers_without_regularized_weights_refuse_regularizers():
    from deeptables_b200 import layers
    with pytest.raises(NotImplementedError, match='kernel_regularizer'):
        layers.BatchNormalization(name='bn', beta_regularizer=None, kernel_regularizer='l2')
    layers.BatchNormalization(name='bn', beta_regularizer=None)


def test_dense_records_kernel_regularizer_and_freeze_lists_segments():
    from deeptables_b200 import layers
    from deeptables_b200.deepmodel import _Scope
    scope = _Scope(torch.device('cpu'), 1)
    x = torch.zeros(2, 3)
    with layers.scope_guard(scope):
        scope.param('a/kernel', (3, 2), 'glorot_uniform')
        dense = layers.Dense(5, kernel_regularizer=R.L1L2(0.5, 0.25), name='d')
        kernel = scope.param('d/kernel', (3, 5), dense.kernel_initializer, regularizer=dense.kernel_regularizer)
        scope.param('d/bias', (5,), 'zeros')
        scope.param('e/kernel', (5, 1), 'glorot_uniform', regularizer='l2')
        scope.param('f/kernel', (5, 1), 'glorot_uniform', regularizer=R.L1L2())
    assert kernel.shape == (3, 5) and x.shape == (2, 3)
    assert scope.regularizers == {'d/kernel': R.RegSpec(0.5, 0.25), 'e/kernel': R.RegSpec(0.0, 0.01)}
    scope.freeze()
    assert scope.reg_segments == [(6, 15, 0.5, 0.25), (26, 5, 0.0, 0.01)]


def test_dnn_builders_pass_kernel_regularizer():
    """dnn() and custom_dnn_D_A_D_B() hand dnn_params['kernel_regularizer'] to every Dense of the tower."""
    from deeptables_b200 import deepnets, layers
    seen = []
    orig = layers.Dense.__init__

    def spy(self, *a, **k):
        orig(self, *a, **k)
        seen.append(self.kernel_regularizer)

    params = {'hidden_units': ((4, 0, True), (3, 0, False)), 'kernel_regularizer': 'l2'}
    deepnets.Dense.__init__ = spy
    try:
        for fn in (deepnets.dnn, deepnets.custom_dnn_D_A_D_B):
            seen.clear()
            with pytest.raises(RuntimeError, match='inside a DeepModel forward pass'):
                fn(torch.zeros(2, 3), params)
            assert seen == [R.RegSpec(0.0, 0.01)], fn.__name__
            with pytest.raises(NotImplementedError, match='activity'):
                fn(torch.zeros(2, 3), {**params, 'activity_regularizer': 'l1'})
    finally:
        deepnets.Dense.__init__ = orig


@pytest.mark.parametrize('l1,l2', [(0.01, 0.0), (0.0, 0.03), (0.02, 0.05)])
def test_reference_formulas_match_autograd(l1, l2):
    g = torch.Generator().manual_seed(3)
    w = torch.randn(40, 7, generator=g, dtype=torch.float64)
    w[0, :3] = 0.0                                          # sign(0) = 0: TensorFlow's gradient of abs at 0
    x = w.clone().requires_grad_(True)
    loss = l1 * torch.abs(x).sum() + l2 * torch.square(x).sum()
    loss.backward()
    torch.testing.assert_close(reg_ref.reg_loss(w, l1, l2), loss.detach(), rtol=1e-15, atol=0)
    torch.testing.assert_close(reg_ref.reg_grad(w, l1, l2), x.grad, rtol=1e-15, atol=0)
    assert bool((reg_ref.reg_grad(w, l1, 0.0)[0, :3] == 0).all())


def test_regularized_weights_picks_tables_and_tower_kernels():
    state = {'cat_embeddings_all/embeddings_0': 0, 'cat_embeddings_all/embeddings_1': 0, 'dnn_dense_1/kernel': 0,
             'dnn_dense_1/bias': 0, 'dnn_dense_2/kernel': 0, 'task_output/kernel': 0, 'linear/kernel': 0}
    got = reg_ref.regularized_weights(state, R.RegSpec(0.0, 1e-5), R.RegSpec(1e-4, 0.0))
    assert got == {'cat_embeddings_all/embeddings_0': (0.0, 1e-5), 'cat_embeddings_all/embeddings_1': (0.0, 1e-5),
                   'dnn_dense_1/kernel': (1e-4, 0.0), 'dnn_dense_2/kernel': (1e-4, 0.0)}
