"""Table rounds of toon_tp_kernel at the edges of its staging buffers, on the GPU: the documents of
test_toon_table_bounds_cpu.py through cf_toon_host and through the fused cf_run_batch, against the oracle."""
import pytest

from mcp_context_forge_b200 import engine
from mcp_context_forge_b200._native import CF_STAGE_TOON, CF_V_TOON
from oracle import toon_ref
from test_toon_table_bounds_cpu import DOCS
from test_toon_tp_gpu import toon

pytestmark = pytest.mark.gpu


def test_cf_toon_host_at_staging_bounds():
    # each document at several offsets in the packed stream, so that it starts at different positions of the 16-byte grid
    texts = [t for _, t in DOCS for _ in range(4)]
    texts = [(" " * (i % 16)) + t for i, t in enumerate(texts)]
    res, _, _ = toon(texts, 0)
    for t, (st, got) in zip(texts, res):
        assert (got.decode("utf-8") if st == 0 else None) == toon_ref.process_text(t, 0, 1 << 30), t[:120]


def test_run_batch_at_staging_bounds():
    ctx = engine.Context.get()
    texts = [t for _, t in DOCS]
    stream, offs = engine.pack_units([engine.encode_unit(t) for t in texts])
    batch = engine.Batch(ctx, len(stream), len(texts))             # `out` is a view of the batch's pinned buffer: keep the batch alive
    v, out, oo, _ = engine.run_batch(None, batch, stream, offs, CF_STAGE_TOON)
    for i, t in enumerate(texts):
        got = out[int(oo[i]):int(oo[i + 1])].tobytes().decode() if v["flags"][i] & CF_V_TOON else None
        assert got == toon_ref.process_text(t, 0, 1 << 30), t[:120]
