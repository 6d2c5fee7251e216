"""H100-native (sm_90a) implementation of SynergyNet's batched inference hot path.

Public surface mirrors the reference: ``synergynet_b200.model_building.SynergyNet(args)``,
``synergynet_b200.synergy3DMM.SynergyNet()``, ``parse_param_62``, ``ParamsPack``.
"""
__version__ = '0.1.0'
