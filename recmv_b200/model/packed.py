"""The packed weight blob a fused network launch reads, cached on its module."""
import torch


def cached_pack(module, pack):
    """pack() -> the module's packed weight blob, rebuilt (under no_grad) only when a parameter's storage or version
    counter changed: the key is (data_ptr, _version) of every parameter."""
    key = tuple((p.data_ptr(), p._version) for p in module.parameters())
    cache = getattr(module, "_packed_cache", None)
    if cache is None or cache[0] != key:
        with torch.no_grad():
            cache = module._packed_cache = (key, pack())
    return cache[1]
