"""GPU: the range encoder's coding and emitter warps (range_coder.cu, ac_encode_kernel<SPC>) against the CPU oracle.

Every stream is a coding warp that hands batches of 32 records through a ring of ENC_RING shared-memory slots to an
emitter warp, SPC streams per CTA (engine.encoder_streams_per_cta).  For each SPC the bytes and out_len of every
stream must equal oracle.ac.encode on test_gpu_coder_launches' streams: 1 to 5003 symbols (partial last batches, a
ring that wraps up to 40 times), streams that owe runs of more than 31 underflow bits across batch boundaries (the
emitter's sequential fallback) and up to the terminator, and streams of 1-count intervals that fill their slot up to
the 17-bits-per-symbol bound.  The launches hold a stream count of 1, 2 and 3 mod 4, so the last CTA is partial."""
import numpy as np
import pytest
import torch

from tests.test_gpu_coder_launches import _encode_and_pack, streams_for

SPCS = (1, 2, 4)


@pytest.mark.gpu
@pytest.mark.parametrize('spc', SPCS)
@pytest.mark.parametrize('L', (3, 25, 256))
def test_encoder_warps_match_the_oracle(L, spc):
    from l3c_pytorch_b200 import engine as E
    dev = torch.device('cuda')
    ss = streams_for(L)
    assert len(ss) % 4 == 1
    for m in (len(ss), len(ss) - 3, len(ss) - 2):           # 1, 2 and 3 mod 4 streams in the launch
        with E.encoder_streams_per_cta(spc):
            lens, dst, blob, caps = _encode_and_pack(ss[:m], L, dev)
        hb = blob.cpu().numpy()
        for i, s in enumerate(ss[:m]):
            assert lens[i] == len(s.want), (L, spc, m, i, s.kind, s.n)
            assert hb[dst[i]:dst[i] + lens[i]].tobytes() == s.want, (L, spc, m, i, s.kind, s.n)
        assert (lens <= caps).all()
    tail = max(8.0 * len(s.want) / s.n for s in ss if s.kind == 'tail' and s.n >= 1000)
    assert tail < 17.0, tail                               # 1-count intervals: the slot bound holds


@pytest.mark.gpu
def test_encoder_streams_per_cta_knob_selects_the_kernel():
    from l3c_pytorch_b200 import engine as E
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device('cuda')
    ss = streams_for(256)[:9]
    for spc in SPCS:
        # the profiler's record of a launch is not guaranteed: on a busy device a capture can come back without any
        # kernel records.  Such a capture says nothing about the knob, so it is taken again (up to 3 times); any
        # capture that did record the encoder must show the selected variant and no other.
        for attempt in range(3):
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                with E.encoder_streams_per_cta(spc):
                    lens, dst, blob, _ = _encode_and_pack(ss, 256, dev)
                torch.cuda.synchronize()
            names = {e.name for e in prof.events() if 'ac_encode_kernel' in e.name}
            hb = blob.cpu().numpy()
            assert all(hb[dst[i]:dst[i] + lens[i]].tobytes() == s.want for i, s in enumerate(ss))
            if names:
                break
        assert names, (spc, 'no encoder launch recorded in 3 profiler captures')
        assert all('ac_encode_kernel<%d>' % spc in n for n in names), (spc, names)


def test_encoder_streams_per_cta_knob_rejects_other_values():
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200._lib import lib
    for bad in (-1, 3, 5, 8, 64):
        with pytest.raises(RuntimeError, match='streams_per_cta'):
            with E.encoder_streams_per_cta(bad):
                pass
    for spc in (0,) + SPCS:
        assert lib.l3c_set_encoder_streams_per_cta(spc) == 0
    assert lib.l3c_set_encoder_streams_per_cta(0) == 0
