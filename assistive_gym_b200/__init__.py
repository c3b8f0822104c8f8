"""agphys — H100-native batched physics step behind Assistive Gym's env surface (see DESIGN.md)."""
__all__ = ['capi', 'scene', 'sim', 'feeding_batch', 'envs']
