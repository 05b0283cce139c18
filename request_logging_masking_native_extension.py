"""Drop-in for the reference's Rust/PyO3 module of the same name: the gateway loads it with
`importlib.import_module("request_logging_masking_native_extension")`
(/root/reference/mcpgateway/middleware/request_logging_middleware.py:320).  Put the repository root
on PYTHONPATH (or install it) and set `experimental_rust_request_logging_masking_enabled=true`.
The implementation is the GPU path in mcp_context_forge_b200/masking.py."""
from mcp_context_forge_b200.masking import (mask_sensitive_data, mask_sensitive_headers, mask_sensitive_json_bytes,  # noqa: F401
                                             mask_sensitive_json_bytes_batch)

__all__ = ["mask_sensitive_data", "mask_sensitive_headers", "mask_sensitive_json_bytes", "mask_sensitive_json_bytes_batch"]
