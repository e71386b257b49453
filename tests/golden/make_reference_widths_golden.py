"""Golden vectors for columns of different embedding widths (fixed_embedding_dim=False), produced by EXECUTING THE
REFERENCE'S OWN model assembly (DeepModel.__build_model, deepmodel.py:259-317) over tests/golden/tf_shim.py, like
make_reference_golden.py, whose helpers it reuses:

    PYTHONHASHSEED=0 python tests/golden/make_reference_widths_golden.py   ->  tests/golden/reference_widths.npz

* models of the nets that read concat_emb_dense (dnn_nets with and without BN in the tower, dcn_nets, cross_dnn_nets,
  cross_nets next to dnn_nets under stacking_op='concat', a case without continuous columns) at mixed widths: inputs,
  weights, inference and training-mode outputs, as make_model_cases records them;
* for every built-in net, whether the reference's builder raises at those widths.  The shim's Concatenate is torch.cat,
  which restates Keras's Concatenate shape check: every axis but the joined one must agree.

The reference's get_nets orders the nets of a config through set(), so a multi-net config is built in an order that
depends on Python's string hashing; hence PYTHONHASHSEED=0 (each case also records the order it was built in).
tests/test_widths_cpu.py requires the CPU oracle to reproduce these vectors, tests/test_widths_gpu.py the CUDA model.
"""
import importlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import tf_shim  # noqa: E402
from make_reference_golden import CIN_SMALL, REFERENCE_ROOT, Recorder, collect_state, np64  # noqa: E402

WIDTH_VOCAB, WIDTH_DIMS = [7, 20, 90, 300, 5], [4, 8, 12, 16, 3]

WIDTH_MODEL_CASES = [
    ('dnn', dict(nets=['dnn_nets'], dnn_params={'hidden_units': ((16, 0, False), (8, 0, False)), 'activation': 'relu'}),
     WIDTH_VOCAB, WIDTH_DIMS, 3, 'binary', 2),
    ('dnn_bn', dict(nets=['dnn_nets'], dnn_params={'hidden_units': ((16, 0, True), (8, 0, False)), 'activation': 'relu'}),
     WIDTH_VOCAB, WIDTH_DIMS, 3, 'binary', 2),
    ('dcn', dict(nets=['dcn_nets'], dnn_params={'hidden_units': ((16, 0, False), (8, 0, False)), 'activation': 'relu'},
                 cross_params={'num_cross_layer': 2}), WIDTH_VOCAB, WIDTH_DIMS, 3, 'regression', None),
    ('cross_dnn', dict(nets=['cross_dnn_nets'], dnn_params={'hidden_units': ((16, 0, False), (8, 0, False)),
                                                            'activation': 'tanh'}, cross_params={'num_cross_layer': 3}),
     WIDTH_VOCAB, WIDTH_DIMS, 2, 'binary', 2),
    ('cross_concat_dnn', dict(nets=['cross_nets', 'dnn_nets'], stacking_op='concat',
                              dnn_params={'hidden_units': ((16, 0, False), (8, 0, False)), 'activation': 'relu'}),
     WIDTH_VOCAB, WIDTH_DIMS, 3, 'binary', 2),
    ('dnn_no_cont', dict(nets=['dnn_nets'], dnn_params={'hidden_units': ((16, 0, True), (8, 0, False)), 'activation': 'relu'}),
     WIDTH_VOCAB, WIDTH_DIMS, 0, 'multiclass', 3),
    ('dcn_widths4', dict(nets=['dcn_nets'], dnn_params={'hidden_units': ((16, 0, False), (8, 0, False)), 'activation': 'relu'},
                         cross_params={'num_cross_layer': 2}), WIDTH_VOCAB, [20, 8, 12, 4, 16], 3, 'binary', 2),
]

WIDTH_NETS = ['linear', 'cin_nets', 'fm_nets', 'afm_nets', 'opnn_nets', 'ipnn_nets', 'pnn_nets', 'dnn_nets', 'cross_nets',
              'cross_dnn_nets', 'dcn_nets', 'autoint_nets', 'fg_nets', 'fgcnn_cin_nets', 'fgcnn_fm_nets', 'fgcnn_afm_nets',
              'fgcnn_ipnn_nets', 'fgcnn_dnn_nets', 'fibi_nets', 'fibi_dnn_nets']


def _build_reference(deepmodel, conf, task, num_classes, cats, conts):
    dm = deepmodel.DeepModel(task, num_classes, conf, cats, conts)
    return dm._DeepModel__build_model(task=task, num_classes=num_classes, nets=conf.nets, categorical_columns=cats,
                                      continuous_columns=conts, var_len_categorical_columns=None, config=conf)


def make_width_cases(deepmodel, config_mod, metainfo, counter, rec):
    for ci, (case, cfg_kwargs, vocab, dims, n_cont, task, num_classes) in enumerate(WIDTH_MODEL_CASES):
        conf = config_mod.ModelConfig(embedding_dropout=0, dense_dropout=0, fixed_embedding_dim=False, **cfg_kwargs)
        cats = [metainfo.CategoricalColumn(f'c{i}', v, d) for i, (v, d) in enumerate(zip(vocab, dims))]
        conts = [metainfo.ContinuousColumn('input_continuous_all', [f'n{i}' for i in range(n_cont)])] if n_cont else []
        b = 9
        g = np.random.default_rng(500 + ci)
        ids = np.stack([g.integers(0, v, size=b) for v in vocab], axis=1)
        cont = g.normal(size=(b, n_cont))
        outs = {}
        for training in (False, True):
            tf_shim.reset_layers()
            tf_shim.seed(5000 + ci)
            tf_shim.set_training(training)
            tf_shim.feed('input_categorical_vars_all', torch.tensor(ids.astype(np.float32)))
            if n_cont:
                tf_shim.feed('input_continuous_all', torch.tensor(cont, dtype=torch.float64))
            model = _build_reference(deepmodel, conf, task, num_classes, cats, conts)
            outs[training] = np64(model.output)
            state = collect_state(tf_shim.created_layers())
            tf_shim.set_training(False)
        params = {k: (list(v) if isinstance(v, tuple) else v) for k, v in cfg_kwargs.items()}
        params['nets'] = list(conf.nets)
        rec.add(case, 'model', {'config': json.loads(json.dumps(params)), 'vocab': vocab, 'dims': dims, 'n_cont': n_cont,
                                'task': task, 'num_classes': num_classes},
                ids=ids.astype(np.int64), cont=cont.astype(np.float64), out_infer=outs[False], out_train=outs[True],
                **{f'w/{k}': v for k, v in state.items()})
    # which built-in nets the reference builds at these widths
    fg = {'fg_filters': (3, 4), 'fg_heights': (3, 2), 'fg_pool_heights': (2, 2), 'fg_new_feat_filters': (2, 1)}
    raises = []
    for net in WIDTH_NETS:
        conf = config_mod.ModelConfig(embedding_dropout=0, dense_dropout=0, fixed_embedding_dim=False, nets=[net],
                                      fgcnn_params=fg, cin_params=CIN_SMALL)
        cats = [metainfo.CategoricalColumn(f'c{i}', v, d) for i, (v, d) in enumerate(zip(WIDTH_VOCAB, WIDTH_DIMS))]
        conts = [metainfo.ContinuousColumn('input_continuous_all', ['n0', 'n1', 'n2'])]
        g = np.random.default_rng(600)
        tf_shim.reset_layers()
        tf_shim.seed(6000)
        counter._data_.clear()
        tf_shim.feed('input_categorical_vars_all',
                     torch.tensor(np.stack([g.integers(0, v, size=4) for v in WIDTH_VOCAB], axis=1).astype(np.float32)))
        tf_shim.feed('input_continuous_all', torch.tensor(g.normal(size=(4, 3))))
        try:
            _build_reference(deepmodel, conf, 'binary', 2, cats, conts)
            raises.append(False)
        except Exception:                                 # noqa: BLE001 -- any failure of the builder counts
            raises.append(True)
    rec.add('nets_at_mixed_widths', 'refusals', {'nets': WIDTH_NETS, 'vocab': WIDTH_VOCAB, 'dims': WIDTH_DIMS},
            raises=np.array(raises))


def main():
    tf_shim.install(REFERENCE_ROOT)
    config_mod = importlib.import_module('deeptables.models.config')
    metainfo = importlib.import_module('deeptables.models.metainfo')
    deepmodel = importlib.import_module('deeptables.models.deepmodel')
    counter = importlib.import_module('deeptables.utils.counter')
    rec = Recorder()
    make_width_cases(deepmodel, config_mod, metainfo, counter, rec)
    rec.save(os.path.join(HERE, 'reference_widths.npz'))
    print(f'reference_widths.npz: {len(rec.manifest)} cases')


if __name__ == '__main__':
    main()
