"""GPU: batch-invariant SAM-BERT inference.  kt_blstm_ragged against the float64 LSTM restatement of oracle/sambert.py and
against nn.LSTM over a packed sequence; every front_half(per_item=True) result of an utterance in a padded batch equals,
bit for bit, the utterance run alone, on both compute paths, for the plain, NSF, SE and filled-pause (FP) models; TtsServer
admits a round of requests with one front_half call, gives each request the audio it gets when served alone, bit for bit,
and does not synchronise after the admitting step.  The seeded models get non-zero LayerNorm biases, as trained ones have:
a padding row's LayerNorm is its bias, which the encoder's k = 3 convs read at an item's last symbol."""
import pytest
import torch
import torch.nn as nn

import kantts_b200 as K
from conftest import rel_l2
from oracle import sambert as osb
from test_gpu_tts_serve import _models, _requests, _serve
from test_gpu_tts_stream import _exact

pytestmark = [pytest.mark.gpu]
DEV = "cuda"
PATHS = ["ffma", "tc"]


def _path(path):
    return _exact() if path == "ffma" else torch.no_grad()


# ---- kt_blstm_ragged ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [128, 40])
def test_blstm_ragged_matches_float64_and_packed_lstm(H):
    B, L, C = 6, 23, 48
    lens = torch.tensor([1, L, 7, 16, 2, L - 1])
    torch.manual_seed(0)
    pred = K.sambert.VarFsmnRnnNARPredictor(C, 11, 1, C, 16, 0.0, 0, H).to(DEV).eval()
    x = torch.randn(B, L, C, generator=torch.Generator().manual_seed(1))
    masks = torch.arange(L)[None, :] >= lens[:, None]
    with torch.no_grad(), _exact():
        got = pred.blstm_infer(x.to(DEV), masks.to(DEV)).cpu()
        packed = nn.utils.rnn.pack_padded_sequence(x.to(DEV), lens, batch_first=True, enforce_sorted=False)
        ref32, _ = nn.utils.rnn.pad_packed_sequence(pred.blstm(packed)[0], batch_first=True, total_length=L)
    sd = {k: v.detach().double().cpu() for k, v in pred.state_dict().items()}
    ref64 = osb.lstm(x.double(), osb._SD(sd), "blstm", 1, True, lens)
    assert got.shape == (B, L, 2 * H)
    assert torch.equal(got[masks], torch.zeros_like(got[masks]))          # rows >= len are exact zeros
    assert rel_l2(got, ref64) < 2e-5, rel_l2(got, ref64)
    assert rel_l2(got, ref32.cpu()) < 2e-5, rel_l2(got, ref32.cpu())
    # each item equals itself run alone at its own length
    with torch.no_grad(), _exact():
        for b in range(B):
            n = int(lens[b])
            one = pred.blstm_infer(x[b:b + 1, :n].to(DEV)).cpu()
            assert torch.equal(one[0], got[b, :n]), b


# ---- front_half invariance ------------------------------------------------------------------------------------------------
LENS = [9, 4, 7, 2, 9, 5, 8, 1]


def _layernorm_biases(am, seed=5):
    """Give every LayerNorm of a seeded model a non-zero bias (the golden FP model has them already)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in am.modules():
            if isinstance(m, nn.LayerNorm):
                m.bias.copy_(0.2 * torch.randn(m.bias.shape, generator=g))
    return am


def _fp_model(golden, cfg=None):
    """The golden filled-pause SAM-BERT (its LayerNorm biases are non-zero); with ``cfg`` (a post-net of another depth) the
    golden weights of every parameter whose shape matches, the rest seeded."""
    g = golden("sambert_fp_small_infer")
    torch.manual_seed(1234)
    am = K.KanTtsSAMBERT(cfg or g.cfg)
    own = am.state_dict()
    am.load_state_dict({k: v for k, v in g.group("sd/").items() if k in own and own[k].shape == v.shape},
                       strict=cfg is None)
    am = am.to(DEV).eval()
    am.fp_dict = {int(k): v.to(DEV) for k, v in g.group("fp_dict/").items()}
    return am


def _variant(golden, name):
    """-> (eval model, requests [(ling, emotion, speaker, length) with a batch dimension of 1])."""
    from golden.make_batch import make_sambert_batch
    if name == "fp":
        cfg, am = golden("sambert_fp_small_infer").cfg, _fp_model(golden)
    elif name == "se":
        from test_gpu_sambert_se import _se_models
        cfg, am, _ = _se_models(golden)
        _layernorm_biases(am)
    else:
        cfg, am, _ = _models(golden, num_mels=82 if name == "nsf" else None)
        _layernorm_biases(am)
    b = make_sambert_batch(dict(cfg, speaker=cfg.get("speaker", 1)), B=len(LENS), L=max(LENS),
                           gen=torch.Generator().manual_seed(31))
    reqs = []
    for i, m in enumerate(LENS):
        spk = b["inputs_speaker"][i:i + 1, :m]
        if name == "se":
            spk = torch.randn(1, 1, cfg["speaker_units"], generator=torch.Generator().manual_seed(40 + i)).expand(1, m, -1)
        reqs.append((b["inputs_ling"][i:i + 1, :m], b["inputs_emotion"][i:i + 1, :m], spk.contiguous(), torch.tensor([m])))
    return am, reqs


def _front(am, reqs):
    inputs = K.infer.pad_requests(reqs)
    return am.front_half(*(t.to(DEV) for t in inputs), per_item=True)


BATCHES = [list(range(k)) for k in range(1, 9)] + [[5, 2, 7, 0, 3, 6], [3, 0], [7, 4], [1, 6, 1]]


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("variant", ["plain", "nsf", "se", "fp"])
def test_front_half_is_batch_invariant(golden, variant, path):
    am, reqs = _variant(golden, variant)
    r = am.mel_decoder.r
    with _path(path), torch.no_grad():
        alone = [_front(am, [q]) for q in reqs]
        if variant == "fp":                            # the model inserts pauses, not in every utterance
            assert any(int(a["inter_lengths"][0]) > m for a, m in zip(alone, LENS))
        for batch in BATCHES:
            f = _front(am, [reqs[i] for i in batch])
            for j, i in enumerate(batch):
                a = alone[i]
                n_sym, n = int(a["inter_lengths"][0]), int(a["lr_len"][0])
                steps = a["memory"].shape[1]
                assert steps == -(-n // r)
                where = (variant, path, batch, i)
                assert torch.equal(f["lr_len"][j], a["lr_len"][0]), where
                assert torch.equal(f["band_width_rows"][j], a["band_width_rows"][0]), where
                assert torch.equal(f["memory"][j, :steps], a["memory"][0]), where
                for k in ("log_dur_p", "pitch_p", "energy_p"):
                    assert torch.equal(f[k][j, :n_sym], a[k][0, :n_sym]), (k,) + where


# ---- server ---------------------------------------------------------------------------------------------------------------
def _count_front_half(am):
    calls = []
    inner = am.front_half

    def counted(*a, **kw):
        calls.append(a[0].shape[0])
        return inner(*a, **kw)

    am.front_half = counted
    return calls


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("kind", ["plain", "nsf", "lookahead", "fp"])
def test_server_admits_a_round_with_one_front_half_call(golden, kind, path):
    cfg, am, gen = _models(golden, num_mels=82 if kind == "nsf" else None, nsf=kind == "nsf")
    _layernorm_biases(am)
    if kind == "fp":                                   # post-net delay 3 = r, as the other served models
        cfg = dict(golden("sambert_fp_small_infer").cfg, postnet_fsmn_num_layers=3)
        am = _fp_model(golden, cfg)
    if kind == "lookahead":
        torch.manual_seed(7)
        gen = K.Generator(in_channels=cfg["num_mels"], channels=32, upsample_scales=[4, 2], upsample_kernal_sizes=[8, 4],
                          resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3], [1, 3]], causal=False).to(DEV).eval()
    reqs = _requests(cfg, 5)
    kw = dict(slots=4, chunk_steps=3, max_steps=48, nsf_f0=("mean_std", 180.0, 40.0) if kind == "nsf" else None,
              allow_lookahead=kind == "lookahead")
    seeds = [101 + i for i in range(len(reqs))] if kind == "nsf" else None
    with _path(path), torch.no_grad():
        server = K.TtsServer(am, gen, **kw)
        calls = _count_front_half(am)
        # four requests before the first step fill the four slots in one admission; the fifth waits for a free slot
        got = _serve(server, reqs, [0, 0, 0, 0, 1], seeds)
        assert calls[0] == 4 and len(calls) == 2 and calls[1] == 1, calls
        del am.front_half
        for i in range(len(reqs)):
            one = _serve(K.TtsServer(am, gen, **kw), [reqs[i]], [0], None if seeds is None else [seeds[i]])[0]
            assert torch.equal(got[i], one), (kind, path, i)


def test_server_does_not_synchronise_after_a_batched_admission(golden):
    cfg, am, gen = _models(golden)
    reqs = _requests(cfg, 4)
    server = K.TtsServer(am, gen, slots=4, chunk_steps=2, max_steps=48)
    for r in reqs:
        server.submit(*r)
    calls = _count_front_half(am)
    with torch.no_grad():
        server.step()                                  # admits all four in one front_half call
        assert calls == [4]
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            pieces = []
            while not server.idle:
                pieces += server.step()[0]
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert {rid for rid, _, _ in pieces} == {0, 1, 2, 3}
