"""Engine.forward_events decides its mode once, on the host, before any device work (dagr_b200.engine.resolve_mode).

Each caller's combination of arguments resolves to its sort form, taps form and overlap / capture flags, and every
combination the engine refuses raises ValueError from the resolver, which needs no GPU."""
from types import SimpleNamespace

import pytest
import torch

from dagr_b200.engine import Engine, _overlaps, resolve_mode

B, N = 2, 1000
RING = torch.zeros(8, dtype=torch.int32)
RINGS = torch.zeros((3, 8), dtype=torch.int32)
TAB = torch.zeros(8, dtype=torch.int32)
STATE = object()


def _feats(dtype=torch.float32, n=B):
    fmt = torch.channels_last if dtype == torch.bfloat16 else torch.contiguous_format
    return [torch.zeros(n, c, 8, 8, dtype=dtype).contiguous(memory_format=fmt) for c in (16, 64, 64, 128, 256)]


def _outs(n=B):
    return {k + "_output": [torch.zeros(n, c, 4, 4), torch.zeros(n, c, 2, 2)] for k, c in (("cls", 2), ("reg", 4), ("obj", 1))}


def _flags(m):
    return m.sort, m.streams, m.state, m.min_idx, m.overlap, m.capture, m.fixed


@pytest.mark.parametrize("overlap", [False, True])
def test_plain_batches(overlap):
    """DAGR.forward_decoded and PipelinedDetector: events-only, and with taps in either format."""
    m = resolve_mode(B, N, overlap=overlap)
    assert _flags(m) == ("batch", 1, None, 0, overlap, True, False) and m.taps is None and m.ring is None
    for dtype, sfx in ((torch.float32, ""), (torch.bfloat16, "_bf16")):
        feats, outs = _feats(dtype), _outs()
        m = resolve_mode(B, N, feats, outs, overlap=overlap)
        # the serial hybrid forward stays eager; the overlapped one is captured
        assert _flags(m) == ("batch", 1, None, 0, overlap, overlap, False)
        t = m.taps
        assert t.feats is feats and t.outs is outs and t.fmt == dtype and t.sfx == sfx
        assert t.planes is None and not t.live and t.state is None and t.min_idx == 0


@pytest.mark.parametrize("profiling,use_graphs", [(True, True), (False, False), (True, False)])
def test_timing_or_no_graphs_runs_serial_and_eager(profiling, use_graphs):
    for image in (False, True):
        m = resolve_mode(B, N, *((_feats(), _outs()) if image else ()), overlap=True, profiling=profiling,
                         use_graphs=use_graphs)
        assert not m.overlap and not m.capture


@pytest.mark.parametrize("overlap,profiling,use_graphs", [(o, p, g) for o in (False, True) for p in (False, True)
                                                          for g in (False, True)])
def test_next_slot_uses_the_overlap_of_a_plain_forward(overlap, profiling, use_graphs):
    eng = SimpleNamespace(overlap=overlap, prof={} if profiling else None, use_graphs=use_graphs, _slot=1, _done=[None, "ev"])
    ov = resolve_mode(B, N, overlap=overlap, profiling=profiling, use_graphs=use_graphs).overlap
    assert ov == _overlaps(overlap, profiling, use_graphs) == (overlap and not profiling and use_graphs)
    assert Engine.next_slot(eng) == ((1, "ev") if ov else None)


@pytest.mark.parametrize("image", [False, True])
def test_streaming_detectors(image):
    """StreamingDetector / FusionStreamingDetector (one ring) and MultiStreamDetector / FusionMultiStreamDetector (S rings,
    a frame plane per camera): never overlapped, never a coarse graph of their own (the detector captures the whole step)."""
    taps = (_feats(), _outs()) if image else ()
    m = resolve_mode(1, N, *taps, ring=RING, overlap=True)
    assert _flags(m) == ("ring", 1, None, 0, False, False, True) and m.ring is RING
    assert m.taps is None if not image else (m.taps.live and m.taps.planes is None)
    planes = dict(image_planes=(TAB, 4)) if image else {}
    m = resolve_mode(2, N, *((_feats(n=4), _outs(4)) if image else ()), ring=RINGS, ring_streams=2, overlap=True, **planes)
    assert _flags(m) == ("rings", 2, None, 0, False, False, True) and m.ring is RINGS
    if image:
        assert m.taps.live and m.taps.planes[0] is TAB and m.taps.planes[1] == 4


@pytest.mark.parametrize("image", [False, True])
def test_incremental_steps(image):
    """AsyncDAGR: the state and n_old of the step; the events-only coarse stack is captured, the hybrid one stays eager."""
    taps = (_feats(), _outs()) if image else ()
    m = resolve_mode(B, N, *taps, stream_state=STATE, n_old=300, overlap=True)
    assert _flags(m) == ("batch", 1, STATE, 300, False, not image, True)
    if image:
        assert m.taps.state is STATE and m.taps.min_idx == 300 and not m.taps.live and m.taps.planes is None
    assert resolve_mode(B, N, n_old=300).min_idx == 0                 # n_old means nothing without a state


@pytest.mark.parametrize("overlap", [False, True])
def test_sequence_windows(overlap):
    """SequenceDetector: a frame plane per window of a plain batch; serial and eager.  Its events-only blocks are plain
    batches and overlap when the engine does."""
    m = resolve_mode(6, N, _feats(n=3), _outs(3), image_planes=(TAB, 1), overlap=overlap)
    assert _flags(m) == ("batch", 1, None, 0, False, False, False)
    assert m.taps.planes == (TAB, 1) and not m.taps.live and m.taps.state is None
    assert resolve_mode(6, N, overlap=overlap).overlap == overlap


@pytest.mark.parametrize("kw,match", [
    (dict(ring_streams=2), "needs a ring control block"),
    (dict(ring=RINGS, ring_streams=3), "B == ring_streams"),
    (dict(B=2, N=N + 1, ring=RINGS, ring_streams=2), "N a multiple"),
    (dict(image_planes=(TAB, 1)), "needs image_feats and image_outs"),
    (dict(image_feats=_feats(), image_planes=(TAB, 1)), "needs image_feats and image_outs"),
    (dict(image_feats=_feats(), image_outs=_outs(), image_planes=(TAB, 1), keep_node_features=True), "keep_node_features"),
    (dict(image_feats=_feats()[:1] + _feats(torch.bfloat16)[1:]), "expected all float32 or all bfloat16"),
    (dict(image_feats=_feats(torch.float16)), "expected all float32 or all bfloat16"),
    (dict(image_feats=[f.contiguous() for f in _feats(torch.bfloat16)]), "channels_last"),
    (dict(stream_state=STATE, ring=RING), "stream_state with a ring"),
    (dict(stream_state=STATE, ring=RINGS, ring_streams=2), "stream_state with a ring"),
    (dict(stream_state=STATE, image_feats=_feats(), image_outs=_outs(), image_planes=(TAB, 1)),
     "stream_state with image_planes"),
])
def test_refusals(kw, match):
    kw = dict(dict(B=B, N=N), **kw)
    with pytest.raises(ValueError, match=match):
        resolve_mode(**kw)
