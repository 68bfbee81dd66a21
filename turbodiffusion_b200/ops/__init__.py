# Mirror of turbodiffusion/ops/__init__.py:1-2
from .core import int8_linear, int8_quant, rmsnorm, layernorm
from .core import Int8Linear, FastRMSNorm, FastLayerNorm
from .core import (fast_rmsnorm, fast_layernorm, layernorm_modulate, layernorm_modulate_quant, gate_residual,
                   rope_interleaved, rmsnorm_rope, int8_linear_prequant, wan_rope_angles, gate_residual_stats,
                   layernorm_modulate_quant_from_stats, dense_attention, dense_attention_jvp)
