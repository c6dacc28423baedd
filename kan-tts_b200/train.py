"""The HiFi-GAN train step and its data-parallel gradient exchange.

``GanStep.step`` follows ``GAN_Trainer.train_step`` (KAN-TTS kantts/train/trainer.py:469-589)
statement for statement -- generator phase (mel + adversarial + feature-matching value), Adam,
then the discriminator phase on a re-generated ``y_`` -- with two scheduling changes that do not
alter any result (SURVEY.md section 3.1 / 8e).  With a PQMF in the model (a multi-band generator) both phases
synthesise the full band from the generator's sub-bands, and the sub-band STFT loss compares them with the PQMF analysis
of the real waveform (trainer.py:476-505, 559-562).  The scheduling changes:
  * the discriminators' weight gradients of the GENERATOR phase are never computed nor reduced:
    the reference computes, all-reduces and then zeroes them (trainer.py:577-578);
  * losses are kept as device tensors; ``.item()`` is only called by ``losses_to_float``.

Launch overhead: one step is ~2500 kernel launches from Python.  ``GanStep(..., cuda_graph=True)``
captures the step into two CUDA graphs (generator fwd/bwd | no-grad generator fwd + discriminator fwd/bwd),
split at the gradient exchanges (the Adam steps stay eager between them), and replays them -- "CUDA streams
and graphs instead of a tracing compiler".  The captured work is identical to the eager step.

Multi-GPU (one process per GPU, ``torch.distributed`` NCCL over NVLink/NVSwitch): the batch is
sharded by utterance, replicas are identical, and the only exchange is the gradient all-reduce
(mean) -- replacing the three DistributedDataParallel wrappers of kantts/models/__init__.py:71-84.
Gradients of each model live in one flat fp32 buffer (``.grad`` tensors are views into it), so the
exchange is ONE in-place NCCL all-reduce per model per phase with no packing copies.
"""
import os

import torch
import torch.distributed as dist

from . import ops


class FlatGrads:
    """Owns a flat fp32 gradient buffer for a module; every parameter's ``.grad`` is a view."""

    def __init__(self, module, direct=True):
        self.params = [p for p in module.parameters() if p.requires_grad]
        n = sum(p.numel() for p in self.params)
        dev = self.params[0].device
        self.flat = torch.zeros(n, device=dev, dtype=torch.float32)
        off = 0
        for p in self.params:
            p.grad = self.flat[off:off + p.numel()].view_as(p)
            off += p.numel()
            if direct:      # the conv backward kernels accumulate straight into these views (ops.mark_direct_grad)
                ops.mark_direct_grad(p)

    def zero(self):
        self.flat.zero_()

    def all_reduce_mean(self, group=None):
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group)
            self.flat.div_(dist.get_world_size(group))

    def set_requires_grad(self, flag):
        for p in self.params:
            p.requires_grad_(flag)


def invalidate_weight_caches(modules):
    """Forget every prepared (kernel-layout) weight of ``modules``, so that the next forward re-runs kt_weight_prepare /
    kt_weight_pack_tc (in place, into the same persistent buffers).  A CUDA-graph step calls it before a capture, so that the
    graph re-prepares the weights its eager optimizer step changed."""
    for m in modules:
        for sub in m.modules():
            c = getattr(sub, "_cache", None)
            if isinstance(c, ops.PreparedWeight):
                c.key = None


class GanStep:
    """model = {"generator": G, "discriminator": {name: D}}, optimizer / scheduler dicts of the same
    shape and ``criterion`` as built by the reference's builders (or this package's)."""

    def __init__(self, model, optimizer, scheduler, criterion, config, skip_unused_d_grads=True, cuda_graph=False,
                 graph_warmup=3, pair_discriminators=True, reuse_real_half=True):
        if criterion.get("subband_stft_loss", None) and model.get("pqmf", None) is None:
            raise ValueError("GanStep: the sub-band STFT loss needs a PQMF in the model (a multi-band generator)")
        self.model, self.optimizer, self.scheduler = model, optimizer, scheduler
        self.criterion, self.config = criterion, config
        self.skip_unused_d_grads = skip_unused_d_grads
        # run each discriminator ONCE per phase on the (generated, real) pair as a batch of 2B (forward_pair)
        self.pair_discriminators = pair_discriminators
        # the discriminators' forward on the REAL waveforms is the same computation in both phases (same weights, same input):
        # the generator phase records it, the discriminator phase reuses it (ops.pair_state); spectral-normed scales excluded
        self.reuse_real_half = reuse_real_half
        self._pair_recorded = False
        self.g_grads = FlatGrads(model["generator"])
        self.d_grads = {k: FlatGrads(m) for k, m in model["discriminator"].items()}
        self.steps = 1
        self.cuda_graph = cuda_graph
        self.graph_warmup = graph_warmup
        self._graphs = None
        self._eager_done = 0
        self._static = None
        self._log = {}

    # ---- the three segments (split at the two gradient exchanges) -----------------------------------------
    def _g_active(self):
        return self.steps >= self.config.get("generator_train_start_steps", 0)

    def _d_active(self):
        return self.steps > self.config["discriminator_train_start_steps"]

    def _seg_generator(self, y, x):
        """generator forward, losses, backward (trainer.py:473-546)"""
        cfg, crit, model, log = self.config, self.criterion, self.model, self._log
        # the discriminators' weights changed at the end of the previous step: re-prepare them on side streams while
        # the generator runs
        pre = self._prefetch(list(model["discriminator"].values()), y) if self._d_active() else None
        y_ = model["generator"](x)
        self._prefetch_join(pre)
        pqmf = model.get("pqmf", None)
        if pqmf is not None:                                   # the full band from the sub-bands (trainer.py:476-479)
            y_mb_ = y_
            y_ = pqmf.synthesis(y_mb_)
        gen_loss = 0.0
        if crit.get("stft_loss", None):
            sc_loss, mag_loss = crit["stft_loss"](y_, y)
            gen_loss = gen_loss + (sc_loss + mag_loss) * crit["stft_loss"].weights
            log["spectral_convergence_loss"], log["log_stft_magnitude_loss"] = sc_loss, mag_loss
        if crit.get("subband_stft_loss", None):               # trainer.py:496-507: halves the losses so far, unweighted
            gen_loss = gen_loss * 0.5
            sub_sc_loss, sub_mag_loss = crit["subband_stft_loss"](y_mb_, pqmf.analysis(y))
            gen_loss = gen_loss + 0.5 * (sub_sc_loss + sub_mag_loss)
            log["sub_spectral_convergence_loss"], log["sub_log_stft_magnitude_loss"] = sub_sc_loss, sub_mag_loss
        if crit.get("mel_loss", None):
            mel_loss = crit["mel_loss"](y_, y)
            gen_loss = gen_loss + mel_loss * crit["mel_loss"].weights
            log["mel_loss"] = mel_loss
        if self._d_active():
            if self.skip_unused_d_grads:
                for fg in self.d_grads.values():
                    fg.set_requires_grad(False)
            adv_loss = 0.0
            fmap_lst_ = []
            want_fm = bool(crit.get("feat_match_loss", None))
            paired = self._can_pair() and want_fm
            fmap_lst = []
            for name, disc in model["discriminator"].items():
                if paired:
                    # disc(y_) [with grad] and the no_grad disc(y) of trainer.py:527-531 as one batch: only the
                    # first B items (y_) carry gradient, the real half is returned detached
                    with ops.grad_items(y_.shape[0]), ops.pair_state("record" if self.reuse_real_half else None):
                        (p_, fmap_), (_, fmap) = disc.forward_pair(y_, y, detach_b=True)
                    self._pair_recorded = self.reuse_real_half
                    fmap_lst.append(fmap)
                else:
                    p_, fmap_ = disc(y_)
                fmap_lst_.append(fmap_)
                adv_loss = adv_loss + crit["generator_adv_loss"](p_)
            gen_loss = gen_loss + adv_loss * crit["generator_adv_loss"].weights
            log["adversarial_loss"] = adv_loss
            if want_fm:
                if not paired:
                    for name, disc in model["discriminator"].items():
                        with torch.no_grad():
                            p, fmap = disc(y)
                            fmap_lst.append(fmap)
                fm_loss = 0.0
                for fmap_, fmap in zip(fmap_lst, fmap_lst_):          # argument order: trainer.py:535-538
                    fm_loss = fm_loss + crit["feat_match_loss"](fmap_, fmap)
                log["feature_matching_loss"] = fm_loss
                gen_loss = gen_loss + fm_loss * crit["feat_match_loss"].weights
            if self.skip_unused_d_grads:
                for fg in self.d_grads.values():
                    fg.set_requires_grad(True)
        log["generator_loss"] = gen_loss
        self.g_grads.zero()
        gen_loss.backward()
        self._join_streams(y)

    def _seg_gopt(self):
        """generator Adam (trainer.py:547-553)"""
        cfg, model = self.config, self.model
        if self._g_active():
            if cfg["generator_grad_norm"] > 0:
                torch.nn.utils.clip_grad_norm_(model["generator"].parameters(), cfg["generator_grad_norm"])
            self.optimizer["generator"].step()
            self.scheduler["generator"].step()

    def _seg_discriminator(self, y, x):
        """discriminator forward/backward on a re-generated y_ (trainer.py:556-580)"""
        cfg, crit, model, log = self.config, self.criterion, self.model, self._log
        if self._d_active():
            self._prefetch_join(self._prefetch([model["generator"]], y))    # generator weights changed just now
            with torch.no_grad():
                y_ = model["generator"](x)
                if model.get("pqmf", None) is not None:          # trainer.py:559-562
                    y_ = model["pqmf"].synthesis(y_)
            dis_loss = 0.0
            real_t, fake_t = 0.0, 0.0
            for name, disc in model["discriminator"].items():
                if self._can_pair() and self._pair_recorded:
                    # [re-generated | real] like the generator phase's batch: the real half is already in the layers' buffers
                    with ops.pair_state("reuse", y_.shape[0]):
                        (p_, fmap_), (p, fmap) = disc.forward_pair(y_.detach(), y)
                elif self._can_pair():
                    (p, fmap), (p_, fmap_) = disc.forward_pair(y, y_.detach())     # trainer.py:560-561 as one batch
                else:
                    p, fmap = disc(y)
                    p_, fmap_ = disc(y_.detach())
                real_loss, fake_loss = crit["discriminator_adv_loss"](p_, p)
                dis_loss = dis_loss + real_loss + fake_loss
                real_t, fake_t = real_t + real_loss, fake_t + fake_loss
            log["real_loss"], log["fake_loss"], log["discriminator_loss"] = real_t, fake_t, dis_loss
            for fg in self.d_grads.values():
                fg.zero()
            dis_loss.backward()
            self._join_streams(y)

    def _seg_gopt_discriminator(self, y, x):
        self._seg_gopt()
        self._seg_discriminator(y, x)

    @staticmethod
    def _prefetch(modules, t):
        if not t.is_cuda or os.environ.get("KANTTS_B200_PREFETCH", "1") == "0":
            return None
        from . import hifigan
        cur = torch.cuda.current_stream()
        streams = ops.wgrad_pool(t.device)
        for s in streams:
            s.wait_stream(cur)
        for m in modules:
            hifigan.prefetch_weights(m, streams)
        return streams

    @staticmethod
    def _prefetch_join(streams):
        if streams:
            cur = torch.cuda.current_stream()
            for s in streams:
                cur.wait_stream(s)

    def _can_pair(self):
        return self.pair_discriminators and all(hasattr(d, "forward_pair") for d in self.model["discriminator"].values())

    @staticmethod
    def _join_streams(t):
        # parameter gradients accumulated inside the kernels (FlatGrads -> ops.mark_direct_grad) may still be in
        # flight on the side streams of the parallel sub-discriminators / resblocks
        if t.is_cuda:
            from . import hifigan
            hifigan.join_side_streams(t.device)

    def _seg_dopt(self):
        """discriminator Adam (trainer.py:581-589)"""
        cfg, model = self.config, self.model
        if self._d_active():
            if cfg["discriminator_grad_norm"] > 0:
                for m in model["discriminator"].values():
                    torch.nn.utils.clip_grad_norm_(m.parameters(), cfg["discriminator_grad_norm"])
            for key in self.optimizer["discriminator"].keys():
                self.optimizer["discriminator"][key].step()
            for key in self.scheduler["discriminator"].keys():
                self.scheduler["discriminator"][key].step()

    def _eager_step(self, y, x):
        self._log = {}
        self._pair_recorded = False
        if self._g_active():
            self._seg_generator(y, x)
            self.g_grads.all_reduce_mean()
        self._seg_gopt_discriminator(y, x)
        if self._d_active():
            for fg in self.d_grads.values():
                fg.all_reduce_mean()
        self._seg_dopt()
        self.steps += 1
        # hand out detached losses and drop our own references: a caller holding last step's losses must not
        # keep the autograd graph (and its stream-bound AccumulateGrad nodes) alive into a later graph capture
        out = {k: (v.detach() if torch.is_tensor(v) else v) for k, v in self._log.items()}
        self._log = {}
        return out

    def invalidate_weight_caches(self, mods=None):
        """Forget every prepared (kernel-layout) weight of ``mods`` (default: all models), so that the next forward
        re-runs kt_weight_prepare / kt_weight_pack_tc (in place, into the same persistent buffers)."""
        if mods is None:
            mods = [self.model["generator"], *self.model["discriminator"].values()]
        invalidate_weight_caches(mods)

    # ---- CUDA-graph replay -----------------------------------------------------------------------------------
    def _capture(self, y, x):
        """Two CUDA graphs: (generator fwd/losses/bwd) and (no-grad generator fwd + discriminator fwd/bwd).  The
        gradient exchanges and the three Adam steps run eagerly between / after them (a dozen foreach launches each;
        graphs holding the optimizer steps crashed cudaGraphLaunch on the full-size model, profiles/r01_notes.md).
        Each graph keeps its own memory pool; no tensor produced inside one graph is consumed by the other."""
        if not (self._g_active() and self._d_active()):
            raise RuntimeError("GanStep(cuda_graph=True): capture needs both phases active (steps >= start steps)")
        self._static = (y.clone(), x.clone())
        sy, sx = self._static
        self._log = {}
        torch.cuda.synchronize()
        g1, g2 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        # the weight re-preparation must be PART of the graph that first uses a model after its (eager) Adam step:
        # g1 re-prepares the discriminators (updated at the end of the previous step), g2 the generator
        self.invalidate_weight_caches(list(self.model["discriminator"].values()))
        with torch.cuda.graph(g1):
            self._seg_generator(sy, sx)
        self.invalidate_weight_caches([self.model["generator"]])
        with torch.cuda.graph(g2):
            self._seg_discriminator(sy, sx)
        self._graphs = (g1, g2)
        self._log = {k: (v.detach() if torch.is_tensor(v) else v) for k, v in self._log.items()}
        # stream capture only RECORDS the kernels: run the step for real by replaying what was captured
        return self._replay(y, x)

    def _replay(self, y, x):
        sy, sx = self._static
        sy.copy_(y, non_blocking=True)
        sx.copy_(x, non_blocking=True)
        g1, g2 = self._graphs
        g1.replay()
        self.g_grads.all_reduce_mean()
        self._seg_gopt()
        g2.replay()
        for fg in self.d_grads.values():
            fg.all_reduce_mean()
        self._seg_dopt()
        self.steps += 1
        return dict(self._log)

    def step(self, batch):
        """batch = (y (B,1,T) waveform, x (B,80,T/hop) mel) on the device -> dict of loss tensors"""
        y, x = batch
        if not self.cuda_graph:
            return self._eager_step(y, x)
        if self._graphs is not None:
            return self._replay(y, x)
        if self._eager_done < self.graph_warmup:
            # eager warm-up on a side stream (allocator / Adam state / one-time CUDA attribute calls settle)
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                out = self._eager_step(y, x)
            torch.cuda.current_stream().wait_stream(s)
            self._eager_done += 1
            return out
        return self._capture(y, x)


def losses_to_float(log):
    return {k: (float(v) if torch.is_tensor(v) else v) for k, v in log.items()}


def optimizer_builder(model_params, opt_name, opt_params):
    """kantts/models/__init__.py:16-19"""
    return getattr(torch.optim, opt_name)(model_params, **opt_params)


def hifigan_model_builder(config, device, capturable=False, fused_optimizer=None, precision="bf16x3"):
    """kantts/models/__init__.py:28-86 without the DDP wrappers (GanStep reduces the flat gradient
    buffers itself); scheduler = torch MultiStepLR as in the shipped yamls.  A multi-band generator
    (``out_channels`` > 1) gets ``model["pqmf"]``, a PQMF with that many sub-bands and the yaml's ``pqmf`` kwargs.  ``capturable=True`` builds
    the Adam optimizers so that ``GanStep(cuda_graph=True)`` can capture their step.  ``fused_optimizer`` (default: on a
    CUDA device) asks torch for its single-kernel Adam (``fused=True``: the same update and the same ``state_dict`` as the
    reference's foreach Adam, ~4 launches per model instead of ~12 multi-tensor passes; ablation: the three Adam steps
    cost 1.4 ms of a 36 ms step).  ``precision``: the tensor-core precision of every model (hifigan.set_precision)."""
    if fused_optimizer is None:
        fused_optimizer = torch.device(device).type == "cuda"
    from . import hifigan
    model = {"discriminator": {}}
    optimizer = {"discriminator": {}}
    scheduler = {"discriminator": {}}
    for name, sect in config["Model"].items():
        if name == "Generator":
            m = hifigan.Generator(**sect["params"]).to(device)
        else:
            m = getattr(hifigan, name)(**sect["params"]).to(device)
        hifigan.set_precision(m, precision)
        oparams = dict(sect["optimizer"].get("params", {}))
        if capturable:
            oparams["capturable"] = True
        if fused_optimizer and sect["optimizer"].get("type", "Adam") in ("Adam", "AdamW") and "fused" not in oparams \
                and "foreach" not in oparams:
            oparams["fused"] = True
        opt = optimizer_builder(m.parameters(), sect["optimizer"].get("type", "Adam"), oparams)
        sch_t = sect["scheduler"].get("type", "StepLR")
        sch = getattr(torch.optim.lr_scheduler, sch_t)(opt, **sect["scheduler"].get("params", {}))
        if name == "Generator":
            model["generator"], optimizer["generator"], scheduler["generator"] = m, opt, sch
        else:
            model["discriminator"][name], optimizer["discriminator"][name], scheduler["discriminator"][name] = m, opt, sch
    out_channels = config["Model"]["Generator"]["params"].get("out_channels", 1)
    if out_channels > 1:
        from .pqmf import PQMF
        model["pqmf"] = hifigan.set_precision(PQMF(subbands=out_channels, **config.get("pqmf", {})).to(device), precision)
    return model, optimizer, scheduler


# ------------------------------------------------------------------------------------------------
# SAM-BERT
# ------------------------------------------------------------------------------------------------


class NoamLR(torch.optim.lr_scheduler.LRScheduler):
    """kantts/train/scheduler.py:25-46: lr = base * sqrt(w) * min(step^-0.5, step * w^-1.5)."""

    def __init__(self, optimizer, warmup_steps):
        self.warmup_steps = warmup_steps
        super().__init__(optimizer)

    def get_lr(self):
        step = max(1, self.last_epoch)
        scale = self.warmup_steps ** 0.5 * min(step ** (-0.5), step * self.warmup_steps ** (-1.5))
        return [base_lr * scale for base_lr in self.base_lrs]


def apply_gradients(loss_total, grads, optimizer, scheduler, grad_clip):
    """The tail of the SAM-BERT and syBERT train steps (Sambert_Trainer.train_step, Textsy_BERT_Trainer.train_step in
    kantts/train/trainer.py) after the loss: zero the flat gradient buffer, backward, the data-parallel all-reduce (mean)
    of that buffer, gradient-norm clipping (``grad_clip`` None: none), the optimizer and the scheduler step."""
    _backward(loss_total, grads)
    _update(grads, optimizer, scheduler, grad_clip)


def _backward(loss_total, grads):
    """Zero the flat gradient buffer, backward into it, and join the weight-gradient streams."""
    grads.zero()
    loss_total.backward()
    ops.join_wgrad_streams(loss_total.device if loss_total.is_cuda else None)


def _update(grads, optimizer, scheduler, grad_clip):
    """The data-parallel all-reduce (mean) of the flat gradient buffer, the clip, the optimizer and the scheduler step."""
    grads.all_reduce_mean()
    if grad_clip is not None:
        torch.nn.utils.clip_grad_norm_(grads.params, grad_clip)
    optimizer.step()
    scheduler.step()


class SambertStep:
    """``Sambert_Trainer.train_step`` (kantts/train/trainer.py:898-1005): teacher-forced forward, MelReconLoss +
    ProsodyReconLoss, backward, gradient-norm clipping, Adam, NoamLR.  Data parallel: the batch is sharded by
    utterance and the only exchange is ONE in-place NCCL all-reduce (mean) of the flat gradient buffer
    (49.2 MB for sambert_24k.yaml) between backward and the clip -- replacing the DistributedDataParallel
    wrapper of kantts/models/__init__.py:120-127.  Losses stay on the device (``losses_to_float`` syncs).

    ``cuda_graph=True``: the forward, the losses and the backward into the flat gradient buffer run as a replayed CUDA graph;
    the all-reduce, the clip, the optimizer and the scheduler stay eager after the replay, as in ``GanStep``.  The collate
    pads each batch to its own longest item, so one graph is captured per distinct batch shape (the shapes and dtypes of
    the batch's tensors, and the model's train() / eval() mode), after ``graph_warmup`` eager steps of that shape; each graph replays from its own static copies
    of the batch, and all graphs share one memory pool (they never run concurrently).  The step never pads a batch: it
    trains on exactly the tensors it is given, as the eager step does.  To bound the number of graphs, pad the batches
    before the step with ``data.pad_sambert_batch`` -- which changes the longest item's results (see there).
    In graph mode the returned losses are copies of the graph's outputs (one device copy each, no host synchronisation), as
    independent of later steps as the eager step's, and ``x_band_width`` / ``h_band_width`` are 0-d int64 device tensors
    (the eager step returns the reference's Python ints).
    Filled-pause (FP) and alignment-search (MAS) models read the host during their forward and are refused."""

    def __init__(self, model, optimizer, scheduler, criterion, grad_clip=1.0, cuda_graph=False, graph_warmup=3):
        if cuda_graph and getattr(model, "fp_enable", False):
            raise ValueError("SambertStep(cuda_graph=True): a filled-pause (FP) model cannot be captured -- the forward "
                             "reads the output length of fp_insert_plan (the spliced symbol count) on the host")
        if cuda_graph and getattr(model, "MAS", False):
            raise ValueError("SambertStep(cuda_graph=True): an alignment-search (MAS) model cannot be captured -- align's "
                             "length validation reads input_lengths / output_lengths on the host")
        self.model, self.optimizer, self.scheduler, self.criterion = model, optimizer, scheduler, criterion
        self.grad_clip = grad_clip
        self.grads = FlatGrads(model)
        self.steps = 0
        # the training epoch the caller's loop is in (Sambert_Trainer.epoch): the warm-up of AttentionBinarizationLoss
        self.epoch = 0
        self.cuda_graph, self.graph_warmup = bool(cuda_graph), int(graph_warmup)
        self._graphs = {}          # batch shape -> (static batch, CUDAGraph, output dict)
        self._warm = {}            # batch shape -> eager steps run
        self._pool = None

    def step(self, batch):
        """batch: dict with the reference collate keys (input_lings, input_emotions, input_speakers,
        valid_input_lengths, valid_output_lengths, mel_targets, durations, pitch_contours, energy_contours),
        tensors already on the model's device; plus ``fp_label`` for a filled-pause (FP) model, whose durations /
        pitch / energy contours are padded to the length with the pauses inserted.  With the two attention losses in the
        criterion (a MAS model, the reference's ``with_MAS``) the batch has ``attn_priors`` (B, T_mel, L), frame-level
        pitch / energy contours and no durations (None or absent): the model finds them by alignment search."""
        if not self.cuda_graph:
            return self._eager_step(batch)
        key = (self.model.training,) + tuple((k, tuple(v.shape), v.dtype) for k, v in sorted(batch.items())
                                             if torch.is_tensor(v))
        entry = self._graphs.get(key)
        if entry is None:
            done = self._warm.get(key, 0)
            if done < self.graph_warmup:
                # eager warm-up of this shape on a side stream (allocator, optimizer state and kernel plans settle)
                self._warm[key] = done + 1
                cur = torch.cuda.current_stream()
                s = torch.cuda.Stream()
                s.wait_stream(cur)
                with torch.cuda.stream(s):
                    out = self._eager_step(batch)
                cur.wait_stream(s)
                return out
            entry = self._capture(key, batch)
        static, graph, out = entry
        for k, v in static.items():
            v.copy_(batch[k], non_blocking=True)
        graph.replay()
        # copies: the graphs share one memory pool, so a later replay of another graph may reuse the outputs' blocks
        res = {k: v.clone() for k, v in out.items()}
        _update(self.grads, self.optimizer, self.scheduler, self.grad_clip)
        self.steps += 1
        return res

    def _capture(self, key, batch):
        static = {k: v.clone() for k, v in batch.items() if torch.is_tensor(v)}
        invalidate_weight_caches([self.model])
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, pool=self._pool):
            out = self._losses(dict(batch, **static))
            _backward(out["TotalLoss"], self.grads)
        if self._pool is None:
            self._pool = graph.pool()
        entry = self._graphs[key] = (static, graph, {k: v.detach() for k, v in out.items()})
        return entry

    def _eager_step(self, batch):
        out = self._losses(batch)
        apply_gradients(out["TotalLoss"], self.grads, self.optimizer, self.scheduler, self.grad_clip)
        self.steps += 1
        return {k: (v.detach() if torch.is_tensor(v) else v) for k, v in out.items()}

    def _losses(self, batch):
        """The forward and the losses -> the step's result dict (TotalLoss still attached to the autograd graph)."""
        fp_label = batch.get("fp_label")
        with_mas = "AttentionCTCLoss" in self.criterion and "AttentionBinarizationLoss" in self.criterion
        res = self.model(
            batch["input_lings"], batch["input_emotions"], batch["input_speakers"], batch["valid_input_lengths"],
            output_lengths=batch["valid_output_lengths"], mel_targets=batch["mel_targets"],
            duration_targets=batch.get("durations"), pitch_targets=batch["pitch_contours"],
            energy_targets=batch["energy_contours"], attn_priors=batch.get("attn_priors") if with_mas else None,
            fp_label=fp_label)
        mel_loss_, mel_loss = self.criterion["MelReconLoss"](
            batch["valid_output_lengths"], batch["mel_targets"], res["dec_outputs"], res["postnet_outputs"])
        dur_loss, pitch_loss, energy_loss = self.criterion["ProsodyReconLoss"](
            res["valid_inter_lengths"], res["duration_targets"], res["pitch_targets"], res["energy_targets"],
            res["log_duration_predictions"], res["pitch_predictions"], res["energy_predictions"])
        loss_total = mel_loss_ + mel_loss + dur_loss + pitch_loss + energy_loss
        fp_loss = None
        if "FpCELoss" in self.criterion:
            fp_loss = self.criterion["FpCELoss"](batch["valid_input_lengths"], res["fp_predictions"], fp_label)
            loss_total = loss_total + fp_loss
        attn_ctc_loss = attn_kl_loss = None
        if with_mas:
            attn_ctc_loss = self.criterion["AttentionCTCLoss"](res["attn_logprob"], batch["valid_input_lengths"],
                                                               batch["valid_output_lengths"])
            attn_kl_loss = self.criterion["AttentionBinarizationLoss"](self.epoch, res["attn_hard"], res["attn_soft"])
            loss_total = loss_total + attn_ctc_loss + attn_kl_loss
        out = {"TotalLoss": loss_total, "mel_loss_": mel_loss_.detach(), "mel_loss": mel_loss.detach(),
               "dur_loss": dur_loss.detach(), "pitch_loss": pitch_loss.detach(),
               "energy_loss": energy_loss.detach(), "x_band_width": res["x_band_width"],
               "h_band_width": res["h_band_width"]}
        if fp_loss is not None:
            out["fp_loss"] = fp_loss.detach()
        if attn_ctc_loss is not None:
            out["attn_ctc_loss"], out["attn_kl_loss"] = attn_ctc_loss.detach(), attn_kl_loss.detach()
        return out


def sambert_model_builder(config, device, fp_dict=None):
    """kantts/models/__init__.py:89-129 without the DDP wrapper: ``config`` is the whole yaml dict with the
    linguistic-unit sizes already merged into ``Model.KanTtsSAMBERT.params`` (bin/train_sambert.py:144-146).
    ``fp_dict`` ({1: en, 2: a, 3: e} linguistic-id tensors) is attached to a filled-pause (FP) model."""
    from . import sambert
    sect = config["Model"]["KanTtsSAMBERT"]
    model = sambert.KanTtsSAMBERT(sect["params"]).to(device)
    if fp_dict is not None:
        model.fp_dict = {k: v.to(device) for k, v in fp_dict.items()}
    return (model,) + _optimizer_and_scheduler(model, sect)


def _optimizer_and_scheduler(model, sect):
    """The optimizer and scheduler of one ``Model.<name>`` yaml section (kantts/models/__init__.py:107-116, 134-143):
    NoamLR is this module's, any other scheduler torch's."""
    opt = optimizer_builder(model.parameters(), sect["optimizer"].get("type", "Adam"),
                            dict(sect["optimizer"].get("params", {})))
    sch_t = sect["scheduler"].get("type", "NoamLR")
    sch_p = sect["scheduler"].get("params", {})
    sch = NoamLR(opt, **sch_p) if sch_t == "NoamLR" else getattr(torch.optim.lr_scheduler, sch_t)(opt, **sch_p)
    return opt, sch


# ------------------------------------------------------------------------------------------------
# syBERT
# ------------------------------------------------------------------------------------------------


class SybertStep:
    """``Textsy_BERT_Trainer.train_step`` (kantts/train/trainer.py:1155-1185): the KanTtsTextsyBERT forward, SeqCELoss over
    the masked positions, ``loss / V`` as the reference divides by the vocabulary size, then the SAM-BERT step's tail
    (``apply_gradients``: backward, the flat-gradient all-reduce that replaces DistributedDataParallel, the clip, Adam,
    NoamLR).  ``step(batch)`` takes the collate's keys (input_lings, valid_input_lengths, targets, bert_masks) on the
    model's device -- ``data.BertMasker`` makes them there -- and returns device tensors {"TotalLoss", "Error"}."""

    def __init__(self, model, optimizer, scheduler, criterion, grad_clip=1.0):
        self.model, self.optimizer, self.scheduler, self.criterion = model, optimizer, scheduler, criterion
        self.grad_clip = grad_clip
        self.grads = FlatGrads(model)
        self.steps = 0

    def step(self, batch):
        res = self.model(batch["input_lings"], batch["valid_input_lengths"])
        logits = res["logits"]
        loss, err = self.criterion["SeqCELoss"](logits, batch["targets"], batch["bert_masks"])
        loss_total = loss / logits.size(-1)
        apply_gradients(loss_total, self.grads, self.optimizer, self.scheduler, self.grad_clip)
        self.steps += 1
        return {"TotalLoss": loss_total.detach(), "Error": err}


def sybert_model_builder(config, device):
    """kantts/models/__init__.py:126-150 without the DDP wrapper: ``config`` is the whole sybert.yaml dict with the
    linguistic-unit sizes merged into ``Model.KanTtsTextsyBERT.params`` (bin/train_sybert.py:129-131)."""
    from . import sambert
    sect = config["Model"]["KanTtsTextsyBERT"]
    model = sambert.KanTtsTextsyBERT(sect["params"]).to(device)
    return (model,) + _optimizer_and_scheduler(model, sect)
