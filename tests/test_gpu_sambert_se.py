"""GPU: the speaker-embedding (SE) SAM-BERT variant.  The model against the golden of the unmodified reference on both
compute paths, its train step, and synthesis from an extracted speaker embedding: through the non-causal NSF-global
generator with synthesize(), and through TtsServer against synthesize() of each request alone."""
import pytest
import torch

import kantts_b200 as K
from conftest import rel_l2
from oracle import dtdnn as od
from test_gpu_sambert import OUT_KEYS, _run_model
from test_gpu_tts_serve import _alone, _serve
from test_gpu_tts_stream import _exact

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("path", ["ffma", "tcgen05"])
def test_sambert_se_small_matches_reference_golden(golden, path):
    g = golden("sambert_se_small")
    ffma = path == "ffma"
    tol_o, tol_g = (1e-5, 2e-4) if ffma else (1e-4, 1e-3)
    model, res, losses = _run_model(g.cfg, g.group("sd/"), g.group("in/"), ffma)
    assert not hasattr(model, "spk_tokenizer")
    for k in OUT_KEYS:
        assert rel_l2(res[k].detach().cpu(), g.t("out/" + k)) < tol_o, (k, rel_l2(res[k].detach().cpu(), g.t("out/" + k)))
    assert torch.equal(res["LR_length_rounded"].cpu(), g.t("out/LR_length_rounded"))
    for got, w in zip(losses, g.t("out/losses").tolist()):
        assert abs(got - w) < 1e-4 * max(1.0, abs(w)), (losses, g.t("out/losses").tolist())
    named = dict(model.named_parameters())
    for k, w in g.group("grad/").items():
        assert named[k].grad is not None, k
        if float(w.abs().max()) > 1e-6:
            assert rel_l2(named[k].grad.cpu(), w) < tol_g, (k, rel_l2(named[k].grad.cpu(), w))


def _se_batch(cfg, gen, B=3, L=10):
    """A collate-style SE batch: every symbol of an utterance carries that utterance's embedding."""
    from golden.make_batch import make_sambert_batch
    b = make_sambert_batch(dict(cfg, speaker=1), B=B, L=L, gen=gen)
    se = torch.randn(B, 1, cfg["speaker_units"], generator=gen)
    return dict(input_lings=b["inputs_ling"], input_emotions=b["inputs_emotion"],
                input_speakers=se.expand(B, L, cfg["speaker_units"]).contiguous(), valid_input_lengths=b["input_lengths"],
                valid_output_lengths=b["output_lengths"], mel_targets=b["mel_targets"], durations=b["duration_targets"],
                pitch_contours=b["pitch_targets"], energy_contours=b["energy_targets"])


def _se_step(cfg, batch, steps, ffma):
    from kantts_b200 import ops, sambert
    torch.manual_seed(1234)
    config = {"Model": {"KanTtsSAMBERT": {"params": cfg, "optimizer": {"type": "Adam", "params": {
        "lr": 1e-3, "betas": [0.9, 0.98], "eps": 1e-9, "weight_decay": 0.0}},
        "scheduler": {"type": "NoamLR", "params": {"warmup_steps": 40}}}}}
    model, opt, sch = K.sambert_model_builder(config, DEV)
    model.train()
    step = K.SambertStep(model, opt, sch, {"MelReconLoss": sambert.MelReconLoss(),
                                           "ProsodyReconLoss": sambert.ProsodyReconLoss()})
    ops.set_force_ffma(ffma)
    try:
        outs = []
        for _ in range(steps):
            torch.manual_seed(77)
            outs.append(step.step(batch))
    finally:
        ops.set_force_ffma(False)
    return model, outs


@pytest.mark.parametrize("ffma", [True, False])
def test_sambert_se_train_step_is_finite_and_deterministic(golden, ffma):
    cfg = golden("sambert_se_small").cfg
    batch = {k: v.to(DEV) for k, v in _se_batch(cfg, torch.Generator().manual_seed(3)).items()}
    assert batch["input_speakers"].dtype == torch.float32
    m1, o1 = _se_step(cfg, batch, 3, ffma)
    m2, o2 = _se_step(cfg, batch, 3, ffma)
    for a, b in zip(o1, o2):
        for k, v in a.items():
            if torch.is_tensor(v):
                assert torch.isfinite(v).all(), k
                assert torch.equal(v, b[k]), k
    for (n, p), (_, q) in zip(m1.named_parameters(), m2.named_parameters()):
        if "emb" not in n and "tokenizer" not in n:
            assert torch.equal(p, q), n


def _se_models(golden, num_mels=None):
    """A small seeded SE SAM-BERT taking 192-d embeddings (about 3.5 frames per symbol) and a seeded D-TDNN."""
    g = golden("sambert_small_infer")
    cfg = dict({k: v for k, v in g.cfg.items() if k != "speaker"}, postnet_fsmn_num_layers=3, SE=True,
               speaker_units=192)
    if num_mels:
        cfg["num_mels"] = num_mels
    torch.manual_seed(1234)
    am = K.KanTtsSAMBERT(cfg)
    with torch.no_grad():
        am.variance_adaptor.duration_predictor.fc.bias.fill_(1.5)
    torch.manual_seed(0)
    se = K.DTDNN()
    od.seed_bn_stats(se, seed=7)
    return cfg, am.to(DEV).eval(), se.to(DEV).eval()


def _embeddings(se, n, seed=21):
    gen = torch.Generator().manual_seed(seed)
    lens = [16000 + 3100 * i for i in range(n)]
    wav = (0.1 * torch.randn(n, max(lens), generator=gen)).to(DEV)
    return K.speaker_embedding(se, wav, lens)                               # (n, 192)


def test_synthesize_with_an_se_model_and_the_nsf_global_noncausal_generator(golden):
    from golden.make_batch import make_sambert_batch
    from test_nsf_stream_cpu import STREAM_CONFIGS
    cfg, am, se = _se_models(golden, num_mels=82)
    B, L = 3, 9
    b = make_sambert_batch(dict(cfg, speaker=1), B=B, L=L, gen=torch.Generator().manual_seed(31), short=3)
    emb = _embeddings(se, B)
    spk = emb[:, None, :].expand(B, L, 192).contiguous()
    torch.manual_seed(7)
    gen = K.Generator(**STREAM_CONFIGS["small_nc"]).to(DEV).eval()
    args = [b["inputs_ling"].to(DEV), b["inputs_emotion"].to(DEV), spk, b["input_lengths"].to(DEV)]
    nsf = dict(nsf_f0=("global", 30.0, 730.0), nsf_seeds=[11, 12, 13])
    with torch.no_grad(), torch.backends.cudnn.flags(enabled=False):
        wavs, res = K.synthesize(am, gen, *args, **nsf)
        other, _ = K.synthesize(am, gen, *args[:2], spk.flip(0), args[3], **nsf)
    assert len(wavs) == B
    for b_, w in enumerate(wavs):
        assert w.shape[0] > 0 and torch.isfinite(w).all(), b_
    # the embedding drives the output: items 0 and 2 swap theirs under the flip
    assert not torch.equal(other[0][: min(other[0].shape[0], wavs[0].shape[0])],
                           wavs[0][: min(other[0].shape[0], wavs[0].shape[0])])


def test_server_request_with_an_embedding_equals_synthesize_alone(golden):
    from golden.make_batch import make_sambert_batch
    cfg, am, se = _se_models(golden)
    torch.manual_seed(7)
    gen = K.Generator(in_channels=cfg["num_mels"], channels=32, upsample_scales=[4, 2], upsample_kernal_sizes=[8, 4],
                      resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3], [1, 3]]).to(DEV).eval()
    lens, arrive = [9, 4, 7, 5], [0, 0, 1, 3]
    b = make_sambert_batch(dict(cfg, speaker=1), B=len(lens), L=max(lens), gen=torch.Generator().manual_seed(31))
    emb = _embeddings(se, len(lens)).cpu()
    reqs = [(b["inputs_ling"][i, :m], b["inputs_emotion"][i, :m], emb[i][None].expand(m, 192).contiguous(), m)
            for i, m in enumerate(lens)]
    with torch.no_grad(), _exact():
        want = [_alone(am, gen, r)[0] for r in reqs]
        got = _serve(K.TtsServer(am, gen, slots=2, chunk_steps=4, max_steps=48), reqs, arrive)
    for i, w in enumerate(want):
        err = rel_l2(got[i].cpu(), w.cpu())
        print(f"SE request {i}: {w.shape[0]} samples, rel err vs synthesize {err:.3e}")
        assert got[i].shape == w.shape and err <= 1e-5
