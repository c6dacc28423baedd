"""CPU checks of TtsServer's batched admission: pad_requests right-pads a round's requests into one KanTtsSAMBERT batch, and
kt_blstm_ragged is exported."""
import torch

from kantts_b200 import _lib
from kantts_b200.infer import pad_requests


def _req(n, units=None, base=0):
    ling = torch.arange(base, base + 4 * n).reshape(1, n, 4)
    emo = torch.full((1, n), base + 1)
    spk = torch.full((1, n), base + 2) if units is None else torch.rand(1, n, units)
    return ling, emo, spk, torch.tensor([n])


def test_pad_requests_right_pads_with_zeros():
    reqs = [_req(3), _req(5, base=7), _req(1, base=3)]
    ling, emo, spk, lengths = pad_requests(reqs)
    assert ling.shape == (3, 5, 4) and emo.shape == (3, 5) and spk.shape == (3, 5)
    assert lengths.tolist() == [3, 5, 1]
    for i, (l, e, s, n) in enumerate(reqs):
        m = int(n)
        assert torch.equal(ling[i, :m], l[0]) and torch.equal(emo[i, :m], e[0]) and torch.equal(spk[i, :m], s[0])
        assert not ling[i, m:].any() and not emo[i, m:].any() and not spk[i, m:].any()
    assert ling.dtype == torch.long and emo.dtype == torch.long


def test_pad_requests_pads_speaker_embedding_rows():
    reqs = [_req(2, units=6), _req(4, units=6)]
    _, _, spk, _ = pad_requests(reqs)
    assert spk.shape == (2, 4, 6) and spk.dtype == torch.float32
    assert torch.equal(spk[0, :2], reqs[0][2][0]) and not spk[0, 2:].any()


def test_single_request_is_unchanged():
    req = _req(4)
    for got, want in zip(pad_requests([req]), req):
        assert torch.equal(got, want)


def test_blstm_ragged_is_exported():
    assert "kt_blstm_ragged" in _lib.PROTOTYPES
