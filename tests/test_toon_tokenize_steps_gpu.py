"""The tokenizer's lane- and step-edge cases of tests/test_toon_tokenize_steps_cpu.py on the GPU: toon_tp_kernel (its step-wise UTF-8
check, its number classification) against the sequential encoder on the same device, through cf_toon_host.
Units are packed one after the other, so their alignments vary."""
import pytest

import test_toon_tokenize_steps_cpu as cases
from mcp_context_forge_b200 import engine

pytestmark = pytest.mark.gpu
SEQ, NOFB = 8, 16


def toon(texts, flags):
    ctx = engine.Context.get()
    stream, offs = engine.pack_units(texts)
    status, got, out_len = engine.toon_host_flags(engine.Batch(ctx, len(stream), len(texts)), stream, offs, flags)
    return [(int(s), g) for s, g in zip(status, got)], status, out_len


def _texts():
    texts = []
    feats = [cases._string(s * 3, at) for s in cases.VALID_UTF8 for at in (0, cases.LONG)]
    feats += [cases._string(b"\xc3\xa9" + s, at) for s in cases.INVALID_UTF8 for at in (0, cases.LONG)]
    feats += [(b"[1," + s + b"]", 3) for s in (b"\xc3\xa9", b"\x80")]
    feats += [(b"[" + d + b",1]", 1 + len(d) // 2) for d in cases.DECIMALS]
    for f, h in feats:
        for base in (cases.STEP, cases.STEP + 5 * 32):
            for k in (1, 2, 3):
                for lead in (0, 5, 13):
                    texts.append(cases._place(f, h, base - k, lead))
    for d in cases.DECIMALS:
        texts.append(b'{"rows":[' + b",".join(b'{"id":%d,"score":%s}' % (i, d) for i in range(40)) + b"]}")
    return texts


def test_tokenizer_edges_equal_sequential():
    texts = _texts()
    seq, _, _ = toon(texts, SEQ)
    tp, _, _ = toon(texts, 0)
    bad = [(t[-80:], x, y) for t, x, y in zip(texts, seq, tp) if x != y]
    assert not bad, bad[:3]


def test_decimal_handover_reason():
    texts = [b'{"rows":[' + b",".join(b'{"id":%d,"score":%s}' % (i, d) for i in range(40)) + b"]}"
             for d in (b"1234567890.123456", b"0.0000123456789012345678")]
    _, st, why = toon(texts, NOFB)
    assert list(st) == [7, 7] and list(why) == [1, 1], (list(st), list(why))
