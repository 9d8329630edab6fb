"""mac-vo_b200: H100-native (sm_90a) hot path for MAC-VO behind its Module plugin interfaces.

Import as `macvo_b200` (alias package at the repo root). See DESIGN.md / INTEGRATION.md.
"""
__version__ = "0.1.0"
