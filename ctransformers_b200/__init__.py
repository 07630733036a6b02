"""ctransformers-b200: H100-native drop-in for ctransformers' quantized eval hot path."""
from .hub import AutoConfig, AutoModelForCausalLM
from .llm import LLM, Config
from .multi import MultiLLM
from .state import SequenceState

__all__ = ["AutoConfig", "AutoModelForCausalLM", "LLM", "Config", "MultiLLM", "SequenceState"]
__version__ = "0.1.0"
