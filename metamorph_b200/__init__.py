"""metamorph_b200 — H100-native (sm_90a) implementation of MetaMorph's data-parallel hot path.

Public surface mirrors the reference package (`metamorph.model.MetaMorphLlamaForCausalLM`,
`metamorph.train.train.train`, `inference.load_metamorph.load_metamorph_model`); see DESIGN.md.
Importing the package never touches the GPU; the C-ABI library is loaded on first kernel call.
"""
__version__ = "0.1.0"


def __getattr__(name):
    if name in ("MetaMorphLlamaForCausalLM", "MetaMorphConfig"):
        from . import model
        return getattr(model, name)
    raise AttributeError(name)
