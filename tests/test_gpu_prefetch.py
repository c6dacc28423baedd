"""Weight prefetch: GanStep re-prepares a model's weights on side streams right after that model's optimizer step
(hifigan.prefetch_weights).  It must cover the weights' next use: until that model's next prefetch, the layers it
re-prepared pack no image, and every image it packed is read by a forward or backward kernel."""
import pytest
import torch

from kantts_b200 import _lib, hifigan
from test_gpu_graph import _build
from test_gpu_parity import DEV, _small_config

pytestmark = [pytest.mark.gpu]

# entry point -> positions of its packed-weight-image arguments (include/kantts_b200.h)
PACKS = {"kt_weight_pack_tc": (3,), "kt_resblock_pack": (2,)}
READS = {"kt_conv1d_fwd_tc": (2,), "kt_conv1d_bwd_data_tc": (3,), "kt_resblock_fwd": (2, 4), "kt_resblock_bwd": (5, 6)}


def test_prefetch_covers_every_image_until_the_next_weight_update(golden, monkeypatch):
    g = golden("trainstep_small")
    step, _ = _build(g, _small_config(g), False)
    batch = (g.t("y").to(DEV), g.t("x").to(DEV))
    for _ in range(2):
        step.step(batch)
    torch.cuda.synchronize()

    lib = _lib.load()
    # ("pack" | "read", image pointer) and, after each prefetch, ("prefetch", model, index of its first event, images it
    # packed, images of the layers it re-prepared)
    events = []
    for table, kind in ((PACKS, "pack"), (READS, "read")):
        for name, pos in table.items():
            def call(*args, _fn=getattr(lib, name), _pos=pos, _kind=kind):
                events.extend((_kind, args[i]) for i in _pos)
                return _fn(*args)
            monkeypatch.setattr(lib, name, call)
    prefetch_weights = hifigan.prefetch_weights

    def prefetch(module, streams):
        convs = [(n, m) for n, m in module.named_modules() if isinstance(m, hifigan._NormedConv)]
        keys = [m._cache.key for _, m in convs]
        n0 = len(events)
        prefetch_weights(module, streams)
        packed = {e[1] for e in events[n0:] if e[0] == "pack"}
        layers = [(n, m) for (n, m), k in zip(convs, keys) if m._cache.key != k]      # the layers it re-prepared
        images = {img.data_ptr(): (n, key) for n, m in layers for key, (img, _) in m._cache.img.items()}
        events.append(("prefetch", id(module), n0, packed, images))

    monkeypatch.setattr(hifigan, "prefetch_weights", prefetch)
    for _ in range(3):
        step.step(batch)
    torch.cuda.synchronize()

    checked, n_packed = set(), 0
    for i, ev in enumerate(events):
        if ev[0] != "prefetch":
            continue
        _, model, _, packed, images = ev
        end = next((e[2] for e in events[i + 1:] if e[:2] == ("prefetch", model)), None)
        if end is None:                       # the model's next use runs past the recorded steps
            continue
        window = events[i + 1:end]            # up to the model's next prefetch
        late = [images[e[1]] for e in window if e[0] == "pack" and e[1] in images]
        assert not late, f"images of prefetched layers packed again before the next weight update: {late}"
        unread = packed - {e[1] for e in window if e[0] == "read"}
        assert not unread, f"{len(unread)} of {len(packed)} prefetched images never read"
        checked.add(model)
        n_packed += len(packed)
    assert len(checked) == 3 and n_packed > 0, (len(checked), n_packed)     # generator + MSD + MPD
