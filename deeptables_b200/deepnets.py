"""Net builders and the nets plug-in registry, name-for-name with the reference
(deeptables/models/deepnets.py): the 9 presets, the builder functions, ``get`` / ``get_nets`` /
``register_nets`` and the 6-argument plug-in signature
``fn(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc)``.

Differences a maintainer should know (INTEGRATION.md):
* builders run define-by-run on torch CUDA tensors each forward pass instead of once on Keras
  symbolic tensors; ``embeddings`` is a lazy ``EmbeddingList`` (ids + table) so the built-in
  builders fuse the gather into their interaction kernels;
* ``get_nets`` keeps the user's order (the reference loses it through ``set()``,
  deepnets.py:486), which only matters for ``stacking_op='concat'``;
* the SURVEY.md 8f rank 3 nets (afm_nets, fibi_nets, fibi_dnn_nets, fg_nets and the fgcnn_* family) run on their own
  kernels (afm.cu, fibinet.cu, fgcnn.cu); var-len columns are not implemented.
"""
from inspect import signature

from . import layers
from .layers import Dense, Concatenate, Flatten, BatchNormalization, Activation, Dropout

WideDeep = ['linear', 'dnn_nets']
DeepFM = ['linear', 'fm_nets', 'dnn_nets']
xDeepFM = ['linear', 'cin_nets', 'dnn_nets']
AutoInt = ['autoint_nets']
DCN = ['dcn_nets']
FGCNN = ['fgcnn_dnn_nets']
FiBiNet = ['fibi_dnn_nets']
PNN = ['pnn_nets']
AFM = ['afm_nets']

# nets that concatenate the field embeddings on axis 1 (or sum each one, linear): with columns of different embedding
# widths (fixed_embedding_dim=False) Keras's Concatenate refuses their input, so DeepModel refuses them at build time
EQUAL_WIDTH_NETS = frozenset(['linear', 'cin_nets', 'fm_nets', 'afm_nets', 'opnn_nets', 'ipnn_nets', 'pnn_nets',
                              'autoint_nets', 'fg_nets', 'fgcnn_cin_nets', 'fgcnn_fm_nets', 'fgcnn_afm_nets',
                              'fgcnn_ipnn_nets', 'fgcnn_dnn_nets', 'fibi_nets', 'fibi_dnn_nets'])


def _concat_embeddings(embeddings, concat_layer_name):
    if embeddings is None or len(embeddings) == 0:
        return None
    if len(embeddings) == 1 and not isinstance(embeddings, layers.EmbeddingList):
        return embeddings[0]
    return Concatenate(axis=1, name=concat_layer_name)(embeddings)


def _shape(x):
    return tuple(x.shape) if x is not None else None


def linear(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """Linear(order-1) interactions (reference deepnets.py:43-66), gather fused."""
    has_emb = embeddings is not None and len(embeddings) > 0
    if not has_emb and dense_layer is None:
        raise ValueError('No input layer exists.')
    x = layers.LinearLogit(name='linear_logit')(embeddings if has_emb else None, dense_layer)
    n_in = (len(embeddings) if has_emb else 0) + (dense_layer.shape[1] if dense_layer is not None else 0)
    model_desc.add_net('linear', (None, n_in), _shape(x))
    return x


def cin_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """Compressed Interaction Network (reference deepnets.py:69-81)."""
    cin_concat = _concat_embeddings(embeddings, 'concat_cin_embedding')
    if cin_concat is None:
        model_desc.add_net('cin', (None), (None))
        return None
    cin_output = layers.CIN(params=config.cin_params)(cin_concat)
    model_desc.add_net('cin', _shape(cin_concat), _shape(cin_output))
    return cin_output


def fm_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """FM pairwise (order-2) interactions (reference deepnets.py:84-96)."""
    concat_embeddings_layer = _concat_embeddings(embeddings, 'concat_fm_embedding')
    if concat_embeddings_layer is None:
        model_desc.add_net('fm', (None), (None))
        return None
    fm_output = layers.FM(name='fm_layer')(concat_embeddings_layer)
    model_desc.add_net('fm', _shape(concat_embeddings_layer), _shape(fm_output))
    return fm_output


def opnn_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """OuterProduct + DNN (reference deepnets.py:110-124)."""
    if embeddings is None or len(embeddings) < 2:
        return None
    op = layers.OuterProduct(config.pnn_params, name='outer_product_layer')(embeddings)
    model_desc.add_net('opnn-outer_product', f'list({len(embeddings)})', _shape(op))
    concat_all = Concatenate(name='concat_opnn_all')([op, concat_emb_dense])
    x_dnn = dnn(concat_all, config.dnn_params, cellname='opnn')
    model_desc.add_net('opnn-dnn', _shape(concat_all), _shape(x_dnn))
    return x_dnn


def ipnn_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """InnerProduct + DNN (reference deepnets.py:127-141)."""
    if embeddings is None or len(embeddings) < 2:
        return None
    ip = layers.InnerProduct(name='inner_product_layer')(embeddings)
    model_desc.add_net('ipnn-inner_product', f'list({len(embeddings)})', _shape(ip))
    concat_all = Concatenate(name='concat_ipnn_all')([ip, concat_emb_dense])
    x_dnn = dnn(concat_all, config.dnn_params, cellname='ipnn')
    model_desc.add_net('ipnn-dnn', _shape(concat_all), _shape(x_dnn))
    return x_dnn


def pnn_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """Inner + outer product + DNN (reference deepnets.py:144-160); both products in one launch."""
    if embeddings is None or len(embeddings) < 2:
        return None
    ip, op = layers.InnerOuterProduct(config.pnn_params, 'pnn_inner_product_layer',
                                      'pnn_outer_product_layer')(embeddings)
    model_desc.add_net('pnn-inner_product', f'list({len(embeddings)})', _shape(ip))
    model_desc.add_net('pnn-outer_product', f'list({len(embeddings)})', _shape(op))
    concat_all = Concatenate(name='concat_pnn_all')([ip, op, concat_emb_dense])
    x_dnn = dnn(concat_all, config.dnn_params, cellname='pnn')
    model_desc.add_net('pnn-dnn', _shape(concat_all), _shape(x_dnn))
    return x_dnn


def dnn_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """MLP tower (reference deepnets.py:163-169)."""
    x_dnn = dnn(concat_emb_dense, config.dnn_params)
    model_desc.add_net('dnn', _shape(concat_emb_dense), _shape(x_dnn))
    return x_dnn


def cross_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """Cross network (reference deepnets.py:172-178)."""
    cross = layers.Cross(params=config.cross_params, name='cross_layer')(concat_emb_dense)
    model_desc.add_net('cross', _shape(concat_emb_dense), _shape(cross))
    return cross


def cross_dnn_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """Cross -> DNN (reference deepnets.py:181-192)."""
    x = concat_emb_dense
    cross = layers.Cross(params=config.cross_params, name='cross_dnn_layer')(x)
    model_desc.add_net('cross_dnn-cross', _shape(x), _shape(cross))
    x_dnn = dnn(cross, config.dnn_params, cellname='cross_dnn')
    model_desc.add_net('cross_dnn-dnn', _shape(cross), _shape(x_dnn))
    return x_dnn


def dcn_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """Cross || DNN (reference deepnets.py:195-207)."""
    x = concat_emb_dense
    cross_out = layers.Cross(params=config.cross_params, name='dcn_cross_layer')(x)
    model_desc.add_net('dcn-widecross', _shape(x), _shape(cross_out))
    dnn_out = dnn(x, config.dnn_params, cellname='dcn')
    model_desc.add_net('dcn-dnn2', _shape(x), _shape(dnn_out))
    stack_out = Concatenate(name='concat_cross_dnn')([cross_out, dnn_out])
    model_desc.add_net('dcn', _shape(x), _shape(stack_out))
    return stack_out


def autoint_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """AutoInt (reference deepnets.py:210-224)."""
    concat_embeddings_layer = _concat_embeddings(embeddings, 'concat_autoint_embedding')
    if concat_embeddings_layer is None:
        model_desc.add_net('autoint', (None), (None))
        return None
    output = concat_embeddings_layer
    for _ in range(config.autoint_params['num_attention']):
        output = layers.MultiheadAttention(params=config.autoint_params)(output)
    output = Flatten()(output)
    model_desc.add_net('autoint', _shape(concat_embeddings_layer), _shape(output))
    return output


def _out_of_scope(name):
    def fn(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
        raise NotImplementedError(f'{name} is outside the hot path of this build (SURVEY.md 8f)')
    fn.__name__ = name
    return fn


def afm_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """Attentional Factorization Machine (reference deepnets.py:99-107)."""
    if embeddings is None or len(embeddings) < 2:
        return None
    afm_output = layers.AFM(params=config.afm_params, name='afm_layer')(embeddings)
    model_desc.add_net('afm', f'list({len(embeddings)})', _shape(afm_output))
    return afm_output


def fg_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """Feature Generation: FGCNN layers over the embedding block, new features + the embeddings (reference deepnets.py:227-261)."""
    scope = layers.current_scope()
    index = scope.next_index('concat_fgcnn_embedding')
    fgcnn_emb_concat = _concat_embeddings(embeddings, f'concat_fgcnn_embedding_{index}')
    if fgcnn_emb_concat is None:
        model_desc.add_net('fgcnn', (None), (None))
        return None
    fgcnn_emb_concat = layers._materialize(fgcnn_emb_concat)
    fg_inputs = fgcnn_emb_concat.unsqueeze(-1)
    p = config.fgcnn_params
    new_features = []
    for filters, width, pool, new_filters in zip(p.get('fg_filters', (14, 16)), p.get('fg_heights', (7, 7)),
                                                 p.get('fg_pool_heights', (2, 2)), p.get('fg_new_feat_filters', (2, 2))):
        fg_inputs, new_feats = layers.FGCNN(filters=filters, kernel_height=width, pool_height=pool,
                                            new_filters=new_filters)(fg_inputs)
        new_features.append(new_feats)
    concat_all_features = Concatenate(axis=1)(new_features + [fgcnn_emb_concat])
    model_desc.add_net('fg', _shape(fgcnn_emb_concat), _shape(concat_all_features))
    return concat_all_features


def fgcnn_cin_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """FGCNN with CIN as deep classifier (reference deepnets.py:264-275)."""
    fg_output = fg_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc)
    if fg_output is None:
        return None
    cin_output = layers.CIN(params=config.cin_params)(fg_output)
    model_desc.add_net('fgcnn-cin', _shape(fg_output), _shape(cin_output))
    return cin_output


def fgcnn_fm_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """FGCNN with FM as deep classifier (reference deepnets.py:278-290)."""
    fg_output = fg_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc)
    if fg_output is None:
        return None
    fm_output = layers.FM(name='fm_fgcnn_layer')(fg_output)
    model_desc.add_net('fgcnn-fm', _shape(fg_output), _shape(fm_output))
    return fm_output


def fgcnn_afm_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """FGCNN with AFM as deep classifier (reference deepnets.py:293-304; the split into F (B, 1, D) tensors that AFM
    concatenates again is skipped)."""
    fg_output = fg_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc)
    if fg_output is None:
        return None
    afm_output = layers.AFM(params=config.afm_params)(fg_output)
    model_desc.add_net('fgcnn-afm', _shape(fg_output), _shape(afm_output))
    return afm_output


def fgcnn_ipnn_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """FGCNN with IPNN as deep classifier (reference deepnets.py:307-324)."""
    fg_output = fg_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc)
    if fg_output is None:
        return None
    inner_product = layers.InnerProduct()(fg_output)
    dnn_input_layers = [Flatten()(fg_output), inner_product]
    if dense_layer is not None:
        dnn_input_layers.append(dense_layer)
    dnn_input = Concatenate()(dnn_input_layers)
    dnn_out = dnn(dnn_input, config.dnn_params, cellname='fgcnn_ipnn')
    model_desc.add_net('fgcnn-ipnn', _shape(fg_output), _shape(dnn_out))
    return dnn_out


def fgcnn_dnn_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """FGCNN with DNN as deep classifier (reference deepnets.py:327-341)."""
    fg_output = fg_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc)
    if fg_output is None:
        return None
    if dense_layer is not None:
        dnn_input = Concatenate()([Flatten()(fg_output), dense_layer])
    else:
        dnn_input = Flatten()(fg_output)
    dnn_out = dnn(dnn_input, config.dnn_params, cellname='fgcnn_dnn')
    model_desc.add_net('fgcnn-ipnn', _shape(fg_output), _shape(dnn_out))
    return dnn_out


def fibi_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """SENET + BilinearInteraction on the original and on the SENET-like embeddings (reference deepnets.py:344-371).
    The reference numbers its layers with a process-wide counter (utils/counter.py); here the index counts the fibi nets of
    THIS model (0 for the first), so that checkpoints do not depend on how many models the process has built."""
    scope = layers.current_scope()
    senet_index = scope.next_index('senet_layer')
    senet_emb_concat = _concat_embeddings(embeddings, f'concat_senet_embedding_{senet_index}')
    if senet_emb_concat is None:
        model_desc.add_net('fibi', (None), (None))
        return None
    p = config.fibinet_params
    senet_pooling_op = p.get('senet_pooling_op', 'mean')
    senet_reduction_ratio = p.get('senet_reduction_ratio', 3)
    bilinear_type = p.get('bilinear_type', 'field_interaction')
    senet_embedding = layers.SENET(pooling_op=senet_pooling_op, reduction_ratio=senet_reduction_ratio,
                                   name=f'senet_layer_{senet_index}')(senet_emb_concat)
    senet_bilinear_out = layers.BilinearInteraction(bilinear_type=bilinear_type,
                                                    name=f'senet_bilinear_layer_{senet_index}')(senet_embedding)
    bilinear_out = layers.BilinearInteraction(bilinear_type=bilinear_type,
                                              name=f'embedding_bilinear_layer_{senet_index}')(senet_emb_concat)
    concat_bilinear = Concatenate(axis=1, name=f'concat_bilinear_{senet_index}')([senet_bilinear_out, bilinear_out])
    model_desc.add_net('fibi', _shape(senet_emb_concat), _shape(concat_bilinear))
    return concat_bilinear


def fibi_dnn_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
    """FiBiNet with DNN as deep classifier (reference deepnets.py:374-386)."""
    if embeddings is None or len(embeddings) <= 1:
        return None
    fibi_output = fibi_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc)
    if dense_layer is None:
        raise ValueError('fibi_dnn_nets concatenates the continuous columns (deepnets.py:382): the model has none')
    dnn_input = Concatenate(name='concat_bilinear_dense')([Flatten(name='flatten_fibi_output')(fibi_output), dense_layer])
    dnn_out = dnn(dnn_input, config.dnn_params, cellname='fibi_dnn')
    model_desc.add_net('fibi-dnn', _shape(fibi_output), _shape(dnn_out))
    return dnn_out


def dnn(x, params, cellname='dnn'):
    """[Dense(use_bias=not bn) -> BN? -> activation -> Dropout?]*  (reference deepnets.py:401-427).
    Without BN the activation is fused into the Dense epilogue kernel."""
    custom_dnn_fn = params.get('custom_dnn_fn')
    if custom_dnn_fn is not None:
        return custom_dnn_fn(x, params, cellname + '_custom')
    hidden_units = params.get('hidden_units', ((128, 0, True), (64, 0, False)))
    activation = params.get('activation', 'relu')
    kernel_initializer = params.get('kernel_initializer', 'he_uniform')
    kernel_regularizer = params.get('kernel_regularizer')
    activity_regularizer = params.get('activity_regularizer')
    if len(hidden_units) <= 0:
        raise ValueError(
            '[hidden_units] must be a list of tuple([units],[dropout_rate],[use_bn]) and at least one tuple.')
    for index, (units, dropout, batch_norm) in enumerate(hidden_units, start=1):
        x = Dense(units, use_bias=not batch_norm, name=f'{cellname}_dense_{index}',
                  activation=None if batch_norm else activation,
                  kernel_initializer=kernel_initializer, kernel_regularizer=kernel_regularizer,
                  activity_regularizer=activity_regularizer)(x)
        if batch_norm:
            x = BatchNormalization(name=f'{cellname}_bn_{index}')(x)
            x = Activation(activation=activation, name=f'{cellname}_activation_{index}')(x)
        if dropout > 0:
            x = Dropout(dropout, name=f'{cellname}_dropout_{index}')(x)
    return x


def custom_dnn_D_A_D_B(x, params, cellname='dnn_D_A_D_B'):
    """Dense(act) -> Dropout -> BN ordering (reference deepnets.py:430-452)."""
    hidden_units = params.get('hidden_units', ((128, 0, True), (64, 0, False)))
    activation = params.get('activation', 'relu')
    kernel_initializer = params.get('kernel_initializer', 'he_uniform')
    kernel_regularizer = params.get('kernel_regularizer')
    activity_regularizer = params.get('activity_regularizer')
    if len(hidden_units) <= 0:
        raise ValueError(
            '[hidden_units] must be a list of tuple([units],[dropout_rate],[use_bn]) and at least one tuple.')
    for index, (units, dropout, batch_norm) in enumerate(hidden_units, start=1):
        x = Dense(units, activation=activation, kernel_initializer=kernel_initializer,
                  kernel_regularizer=kernel_regularizer, activity_regularizer=activity_regularizer,
                  name=f'{cellname}_dense_{index}')(x)
        if dropout > 0:
            x = Dropout(dropout, name=f'{cellname}_dropout_{index}')(x)
        if batch_norm:
            x = BatchNormalization(name=f'{cellname}_bn_{index}')(x)
    return x


custom_nets = {}


def get(identifier):
    """Name or callable -> builder function (reference deepnets.py:455-478)."""
    if identifier is None:
        raise ValueError('identifier can not be none.')
    if isinstance(identifier, str):
        fn = custom_nets.get(identifier)
        if fn is not None:
            return fn
        fn = globals().get(identifier)
        if fn is None or not callable(fn) or identifier.startswith('_'):
            raise ValueError(f'Unknown nets function: {identifier}')
        return fn
    if callable(identifier):
        register_nets(identifier)
        return identifier
    raise TypeError(f'Could not interpret nets function identifier: {repr(identifier)}')


def get_nets(nets):
    str_nets = []
    for net in nets:                      # order kept, duplicates dropped
        name = net if isinstance(net, str) else register_nets(net)
        if name not in str_nets:
            str_nets.append(name)
    return str_nets


def register_nets(nets_fn):
    if not callable(nets_fn):
        raise ValueError('nets_fn must be a valid callable function.')
    if signature(nets_fn) != signature(linear):
        raise ValueError(f'Signature of nets_fn is invalid, except {signature(linear)}  but {signature(nets_fn)}')
    custom_nets[nets_fn.__name__] = nets_fn
    return nets_fn.__name__
