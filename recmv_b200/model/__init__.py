"""Mirror of the reference's `model` package surface used by train.py / infer_fl.py
(model/__init__.py:1 re-exports network.*)."""
from .Embedder import Embedder, get_embedder  # noqa: F401
from .network import ImplicitNetwork, getTmpSdf  # noqa: F401
from .Deformer import CompositeDeformer, LBSkinner, MLPTranslator, batch_rodrigues, initialLBSkinner  # noqa: F401
from .RenderNet import RenderingNetwork_view_norm  # noqa: F401
