"""deeptables_b200 -- H100-native (sm_90a) feature-interaction engine behind the DeepTables surface.

    from deeptables_b200 import deeptable, deepnets
    conf = deeptable.ModelConfig(nets=deepnets.xDeepFM, embedding_dropout=0)
    dt = deeptable.DeepTable(config=conf)
    model, history = dt.fit(df, y, batch_size=65536, epochs=1)

Importing the package loads the sm_90a shared library (deeptables_b200/_native); it raises if the
library has not been built -- there is no CPU fallback.
"""
from . import _native            # noqa: F401  (fails loudly when the extension is missing)
from . import consts, metainfo, layers, deepnets, config, deepmodel
from .config import ModelConfig
from .deepmodel import DeepModel
from . import deeptable as _deeptable_module
from .deeptable import DeepTable

# `deeptable.ModelConfig` / `deeptable.DeepTable` as in `from deeptables.models import deeptable`
deeptable = _deeptable_module
deeptable.ModelConfig = ModelConfig

__version__ = '0.1.0'
__all__ = ['deeptable', 'deepnets', 'deepmodel', 'layers', 'config', 'consts', 'metainfo', 'ModelConfig',
           'DeepModel', 'DeepTable']
