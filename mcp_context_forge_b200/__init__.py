"""mcp_context_forge_b200 — H100-native (sm_90a) implementation of ContextForge's plugin hook-chain
hot path: regex_filter / deny_filter / harmful_content_detector scans, the request_logging_masking
redactor and the toon_encoder, behind the reference's Plugin / PluginManager API.

Host code is Python (like the reference); the data path is hand-written CUDA in libcfgpu.so reached
through ctypes (see include/cfgpu.h).  See DESIGN.md.
"""
__version__ = "0.1.0"
