"""Helpers shared by the checkpoint re-sharding tools."""
import re
from typing import Any, Dict, List, Tuple


def descend(state: Dict[str, Any], namespace: str) -> Dict[str, Any]:
    """Follow ``a/b`` style namespaces into nested state dicts (e.g. Swin-MoE keeps weights under 'model')."""
    for key in [k for k in (namespace or '').split('/') if k]:
        state = state[key]
    return state


def moe_layer_prefixes(state: Dict[str, Any]) -> List[str]:
    """Prefixes (with trailing dot, possibly empty) of every MoE layer recorded in ``state``."""
    return sorted({k[: -len('_num_global_experts')] for k in state if k.endswith('_num_global_experts')})


def expert_param_keys(state: Dict[str, Any], prefix: str) -> List[str]:
    return sorted(k for k in state if k.startswith(prefix + 'experts.'))


def legacy_prefixes(state: Dict[str, Any]) -> List[str]:
    """Layers saved before `_num_global_experts` existed: detected through their `experts.batched_fc1_w` tensor.  (A
    prefix is empty or ends with a dot: a layer's replicated `shared_experts.*` tensors are not a legacy layer.)"""
    out = set()
    for k in state:
        m = re.match(r'^((?:.*\.)?)experts\.[^.]+$', k)
        if m and (m.group(1) + '_num_global_experts') not in state:
            out.add(m.group(1))
    return sorted(out)
