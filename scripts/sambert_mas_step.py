"""Time the alignment-learning (MAS) SAM-BERT train step at sambert_16k_MAS.yaml sizes (batch 16, up to 200 symbols, up
to 1000 frames) against the same model with MAS off on a batch with given durations, and the alignment segment
(attention forward + backward, MAS, forward-sum loss forward + backward) against the reference formulation run through the
oracle on the same GPU tensors: the materialised (B, C, T_mel, T_text) difference tensor, one torch.nn.CTCLoss call per
utterance and the host DP.  Reports torch.cuda.max_memory_allocated of each and whether both gave the same hard
alignments and durations, and the device time of the forward-sum loss kernels alone (kt_attn_ctc_fwd, kt_attn_ctc_bwd)
on the batch's attention log-probabilities.  Prints one JSON line with the card name and power limit.

    python scripts/sambert_mas_step.py [--steps 10] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import kantts_b200 as K  # noqa: E402
from kantts_b200 import sambert, sambert_ops  # noqa: E402
from oracle import sambert_mas as om  # noqa: E402
from test_gpu_sambert_mas import make_mas_batch  # noqa: E402

DEV = "cuda"


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def _event_ms(fn, steps, warmup):
    """Mean device time of ``fn`` between CUDA events over ``steps`` calls, after ``warmup``."""
    for _ in range(warmup):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def _ctc_kernel_ms(lp, in_len, out_len, steps, warmup):
    """Device time of kt_attn_ctc_fwd (with its batch-mean launch) and of kt_attn_ctc_bwd, each called on its own."""
    from kantts_b200 import _lib
    from kantts_b200._lib import ptr
    from kantts_b200.ops import call
    B, Tq, Tk = lp.shape
    n = int(_lib.load().kt_attn_ctc_workspace_bytes(B, Tq, Tk))
    ws = torch.empty(n // 4, device=DEV)
    loss, d_loss, grad = torch.empty(1, device=DEV), torch.ones(1, device=DEV), torch.empty_like(lp)
    il, ol = in_len.to(torch.int32).contiguous(), out_len.to(torch.int32).contiguous()
    fwd = lambda: call("kt_attn_ctc_fwd", ptr(lp), ptr(il, True), ptr(ol, True), ptr(loss), ptr(ws), n, B, Tq, Tk, -1.0)
    bwd = lambda: call("kt_attn_ctc_bwd", ptr(lp), ptr(il, True), ptr(ol, True), ptr(d_loss), ptr(ws), n, ptr(grad), B,
                       Tq, Tk, -1.0)
    fwd_ms = _event_ms(fwd, steps, warmup)
    return fwd_ms, _event_ms(bwd, steps, warmup)


def _step(cfg, batch, mas):
    torch.manual_seed(1234)
    model = sambert.KanTtsSAMBERT(cfg).to(DEV).train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-4, betas=(0.9, 0.98), eps=1e-9)
    crit = {"MelReconLoss": sambert.MelReconLoss(), "ProsodyReconLoss": sambert.ProsodyReconLoss()}
    if mas:
        crit.update(AttentionCTCLoss=sambert.AttentionCTCLoss(), AttentionBinarizationLoss=sambert.AttentionBinarizationLoss())
    step = K.SambertStep(model, opt, K.train.NoamLR(opt, warmup_steps=4000), crit)
    step.epoch = 10
    return lambda: step.step(batch)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sambert_mas_step.py measures on the GPU; no CUDA device found")
    cfg = K.sambert_16k_mas_config()
    batch = {k: (v.to(DEV) if v is not None else None)
             for k, v in make_mas_batch(cfg, torch.Generator().manual_seed(1234)).items()}
    B, L = batch["input_lings"].shape[:2]
    Tm = batch["mel_targets"].shape[1]
    res = {"card": _card(), "batch": B, "symbols": L, "frames": Tm, "steps": args.steps, "warmup": args.warmup}
    res["mas_step_ms"], res["mas_step_peak_mib"] = _time(_step(cfg, batch, True), args.steps, args.warmup)

    # MAS off: the same shapes with given durations (each utterance's frames spread over its symbols, the trailing
    # symbol takes the padding frames) and per-symbol pitch / energy
    il, ol = batch["valid_input_lengths"].cpu(), batch["valid_output_lengths"].cpu()
    dur = torch.zeros(B, L)
    for b in range(B):
        n, t = int(il[b]), int(ol[b])
        dur[b, :n] = t // n
        dur[b, : t % n] += 1
        dur[b, n] = Tm - t
    plain = dict(batch, durations=dur.to(DEV), pitch_contours=torch.rand(B, L, device=DEV),
                 energy_contours=torch.rand(B, L, device=DEV), attn_priors=None)
    res["no_mas_step_ms"], res["no_mas_step_peak_mib"] = _time(_step(dict(cfg, MAS=False), plain, False), args.steps,
                                                              args.warmup)

    C = cfg["num_mels"]
    gen = torch.Generator().manual_seed(7)
    q = (torch.randn(B, Tm, C, generator=gen) * 3).to(DEV).requires_grad_(True)
    k = (torch.randn(B, L, C, generator=gen) * 3).to(DEV).requires_grad_(True)
    prior, in_len, out_len = batch["attn_priors"], batch["valid_input_lengths"], batch["valid_output_lengths"]
    mask = torch.arange(L, device=DEV)[None, :] >= in_len[:, None]
    out = {}

    def kernels():
        soft, lp = sambert_ops.AlignAttnFn.apply(q, k, prior, in_len)
        hard, d = sambert_ops.mas(soft, in_len, out_len)
        loss = sambert_ops.AttnCtcFn.apply(lp, in_len, out_len, -1.0) + K.AttentionBinarizationLoss()(10, hard, soft)
        loss.backward()
        out["kernels"] = (hard, d)

    def reference():
        soft, lp = om.distance_attention(q, k, mask, prior)
        hard = torch.from_numpy(om.b_mas(soft.detach().cpu().numpy(), in_len.cpu().numpy(), out_len.cpu().numpy())).to(DEV)
        loss = om.forward_sum_loss(lp, in_len, out_len) + om.binarization_loss(10, hard, soft)
        loss.backward()
        out["reference"] = (hard, hard.sum(2)[:, 0, :])

    res["align_kernels_ms"], res["align_kernels_peak_mib"] = _time(kernels, args.steps, args.warmup)
    with torch.no_grad():
        _, lp = sambert_ops.AlignAttnFn.apply(q, k, prior, in_len)
    res["attn_ctc_fwd_ms"], res["attn_ctc_bwd_ms"] = _ctc_kernel_ms(lp[:, 0].contiguous(), in_len, out_len,
                                                                    max(20, args.steps), args.warmup)
    res["align_reference_ms"], res["align_reference_peak_mib"] = _time(reference, max(1, args.steps // 5), 1)
    res["hard_alignments_equal"] = torch.equal(out["kernels"][0], out["reference"][0])
    res["durations_equal"] = torch.equal(out["kernels"][1], out["reference"][1])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
