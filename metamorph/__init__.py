"""Drop-in alias package: `import metamorph.model`, `metamorph.train.train`, ... resolve to the H100
implementation (metamorph_b200). Lets reference call sites switch without editing imports."""
from metamorph_b200.model import MetaMorphLlamaForCausalLM  # noqa: F401
