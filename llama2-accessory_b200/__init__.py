"""llama2-accessory_b200: H100-native (sm_90a) quantised decode engine behind LLaMA2-Accessory's
MetaModel / Transformer.forward_inference / fairscale-style parallel-linear surface.

Import as `llama2_accessory_b200` (the directory name carries a hyphen; the repo-root module
`llama2_accessory_b200.py` maps the importable name onto this directory).
"""
from . import _cabi  # noqa: F401


def library_path():
    return _cabi.LIB_PATH


def build(verbose=False):
    from ._build import build as _b
    return _b(verbose=verbose)
