"""CPU checks of streamed text-to-speech (PostNet.streamer, infer.stream_synthesize): a chunk-by-chunk restatement of the
post-net over the oracle's own functions (postnet_stream below) equals the oracle's whole-sequence post-net for every
chunk schedule, ragged batches and both post-net delays; the stream plan's delay, windows and launch count follow from the
shapes; bad models are rejected."""
import pytest
import torch
import torch.nn.functional as F

import kantts_b200 as K
from kantts_b200.sambert import PostNet, PostNetStreamPlan
from oracle import sambert as O

# a reduced-width post-net with the shipped filter and layer count; shift 17 gives rp = 3 per layer (D = 12), shift 0
# gives rp = 20 (D = 80, longer than the utterance: only the flush produces output)
SMALL = dict(num_mels=8, postnet_filter_size=41, postnet_fsmn_num_layers=4, postnet_num_memory_units=16,
             postnet_ffn_inner_dim=24, postnet_dropout=0.1, postnet_shift=17, postnet_lstm_units=8)
T = 30
LENGTHS = [30, 7, 22]                   # ragged; slot 1 is shorter than D = 12
SCHEDULES = {"ones": [1] * T, "threes": [3] * (T // 3), "irregular": [5, 1, 2, 9, 3, 10], "all": [T]}


def postnet_stream(p, cfg, lengths, chunks):
    """The whole-sequence post-net output ``(postnet(dec) + dec)`` masked beyond ``lengths``, restated chunk by chunk with
    the oracle's functions: per FSMN layer the feed-forward net runs on the chunk's rows, the memory block keeps the last
    k - 1 rows of its (masked) input and runs UNPADDED over [history | chunk], so its outputs are the rows rp behind, and
    the residual keeps rp rows; the LSTM steps with its carried state over rows of frame >= 0; ``delay`` padding rows flush
    the last outputs.  A row is padding when its frame lies outside [0, lengths[b]).  -> (output rows, delay)."""
    n, k, shift = cfg["postnet_fsmn_num_layers"], cfg["postnet_filter_size"], cfg["postnet_shift"]
    lp = int(round((k - 1) / 2)) + max(shift, 0)
    rp = int((k - 1) / 2) - max(shift, 0)
    delay = n * rp
    fs = p.sub("fsmn")
    B, M = chunks[0].shape[0], chunks[0].shape[2]
    units = cfg["postnet_num_memory_units"]

    def keep(first, rows):
        a = torch.arange(first, first + rows)[None, :]
        return ((a >= 0) & (a < lengths[:, None])).unsqueeze(-1)

    def tail(x, h):
        return x[:, x.shape[1] - h:]

    hist_ctx = [chunks[0].new_zeros(B, k - 1, units) for _ in range(n)]
    hist_x = [None] + [chunks[0].new_zeros(B, rp, units) for _ in range(1, n)]
    hist_dec = chunks[0].new_zeros(B, delay, M)
    state, outs, a = None, [], 0
    for x in list(chunks) + [chunks[0].new_zeros(B, delay, M)]:
        f = x.shape[1]
        dec = torch.cat([hist_dec, x], 1)
        hist_dec = tail(dec, delay)
        cur, lag = x, 0
        for i in range(n):
            ffn = fs.sub(f"ffn_lst.{i}")
            ctx = O.conv_tl(F.relu(O.conv_tl(cur, ffn.sub("w_1"), 0)), ffn.sub("w_2"), 0) * keep(a - lag, f)
            full = torch.cat([hist_ctx[i], ctx], 1)
            hist_ctx[i] = tail(full, k - 1)
            w = fs[f"memory_block_lst.{i}.conv_dw.weight"]
            mem = F.conv1d(full.transpose(1, 2), w, None, groups=w.shape[0]).transpose(1, 2) + full[:, lp:lp + f]
            mem = mem * keep(a - lag - rp, f)
            if mem.shape[-1] == cur.shape[-1]:
                xf = torch.cat([hist_x[i], cur], 1)
                hist_x[i] = tail(xf, rp)
                mem = mem + xf[:, :f]
            cur, lag = mem, lag + rp
        for t in range(max(0, delay - a), f):                       # output row t is frame a - delay + t
            h, state = O.lstm_step(cur[:, t], p, "lstm", 1, state)
            y = O.linear(h, p.sub("fc")) + dec[:, t]
            outs.append(y.unsqueeze(1) * keep(a - delay + t, 1))
        a += f
    return torch.cat(outs, 1), delay


def _postnet(shift, seed=3):
    torch.manual_seed(seed)
    return PostNet(dict(SMALL, postnet_shift=shift)).eval()


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("shift", [17, 0])
def test_oracle_stream_equals_whole_postnet(shift, schedule):
    cfg = dict(SMALL, postnet_shift=shift)
    pn = _postnet(shift)
    sd = {k: v.detach().double() for k, v in pn.state_dict().items()}
    p = O._SD(sd)
    lengths = torch.tensor(LENGTHS)
    mask = O.length_mask(lengths, T)
    dec = torch.randn(len(LENGTHS), T, cfg["num_mels"], generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    dec = dec.masked_fill(mask.unsqueeze(-1), 0)
    want = (O.postnet(dec, mask, p, cfg) + dec).masked_fill(mask.unsqueeze(-1), 0)
    got, delay = postnet_stream(p, cfg, lengths, list(torch.split(dec, SCHEDULES[schedule], 1)))
    assert delay == PostNetStreamPlan(pn).delay == (12 if shift == 17 else 80)
    assert got.shape == want.shape
    assert float((got - want).abs().max()) <= 1e-10


def _yaml_postnet(**over):
    """PostNet of the shipped sambert yaml values (sambert_16k / 24k / 48k / fp_8k differ only in num_mels here)."""
    return PostNet(dict(K.sambert_24k_config(), **over)).eval()


def test_plan_delay_of_the_shipped_configs():
    assert PostNetStreamPlan(PostNet(K.sambert_24k_config()).eval()).delay == 12
    assert PostNetStreamPlan(PostNet(K.sambert_fp_8k_config()).eval()).delay == 12
    assert PostNetStreamPlan(_yaml_postnet(num_mels=80)).delay == 12           # sambert_16k.yaml
    assert PostNetStreamPlan(_yaml_postnet(num_mels=128)).delay == 12          # sambert_48k.yaml


def test_plan_windows_keep_the_history_their_readers_need():
    plan = PostNetStreamPlan(_yaml_postnet())
    win = {w["name"]: w for w in plan.windows}
    assert [(L["lp"], L["rp"], L["kernel"], L["lag"]) for L in plan.layers] == [(37, 3, 41, 3 * i) for i in range(4)]
    for i in range(4):
        assert win[f"ctx{i}"]["history"] == 40 and win[f"ctx{i}"]["channels"] == 256     # the memory block: k - 1
    # layer 0 reads the 80-channel decoder rows (no residual: 80 != 256); layers 1..3 add their input rp = 3 rows back
    assert [win[f"x{i}"]["history"] for i in (1, 2, 3, 4)] == [3, 3, 3, 0]
    assert win["dec"]["history"] == 12 and win["dec"]["channels"] == 80               # the output Linear's residual
    assert win["gates"]["channels"] == 512 and win["h"]["channels"] == 128
    assert all(win[n]["history"] == 0 for n in ("mid", "gates", "h", "out"))


def test_launches_per_chunk_include_the_output_mask():
    # per FSMN layer: two feed-forward convs + the memory block; LSTM input projection, LSTM, output Linear; one advance;
    # one output mask
    assert PostNetStreamPlan(_yaml_postnet()).launches_per_chunk == 3 * 4 + 3 + 1 + 1
    for layers in (1, 2, 3):
        assert PostNetStreamPlan(PostNet(dict(SMALL, postnet_fsmn_num_layers=layers)).eval()).launches_per_chunk == 3 * layers + 5


def test_plan_rejects_what_it_cannot_stream():
    with pytest.raises(ValueError, match="rp >= 0"):
        PostNetStreamPlan(PostNet(dict(SMALL, postnet_filter_size=5, postnet_shift=3)).eval())
    with pytest.raises(ValueError, match="eval"):
        PostNetStreamPlan(PostNet(SMALL).train())
    with pytest.raises(RuntimeError, match="CUDA"):                            # no CPU fallback
        _postnet(17).streamer(batch=1, max_frames=4, lengths=torch.tensor([4]))


def _models(golden, **gen_over):
    g = golden("sambert_small_infer")
    am = K.KanTtsSAMBERT(g.cfg)
    am.load_state_dict(g.group("sd/"), strict=True)
    gcfg = dict(in_channels=g.cfg["num_mels"], channels=32, upsample_scales=[4, 2], upsample_kernal_sizes=[8, 4],
                resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3], [1, 3]])
    gcfg.update(gen_over)
    torch.manual_seed(7)
    return am.eval(), K.Generator(**gcfg).eval()


def test_stream_synthesize_rejects_bad_models(golden):
    inputs = (torch.zeros(1, 4, 4, dtype=torch.long), torch.zeros(1, 4, dtype=torch.long), torch.zeros(1, 4, dtype=torch.long),
              torch.tensor([4]))
    am, gen = _models(golden)
    with pytest.raises(RuntimeError, match="eval"):
        K.stream_synthesize(am.train(), gen, *inputs)
    am.eval()
    with pytest.raises(RuntimeError, match="eval"):
        K.stream_synthesize(am, gen.train(), *inputs)
    with pytest.raises(ValueError, match="causal"):
        K.stream_synthesize(am, _models(golden, causal=False)[1], *inputs)
    with pytest.raises(ValueError, match="NSF"):
        K.stream_synthesize(am, _models(golden, nsf_params=dict(nb_harmonics=7, sampling_rate=16000))[1], *inputs)
    with pytest.raises(ValueError, match="mel channels"):
        K.stream_synthesize(am, _models(golden, in_channels=80)[1], *inputs)
