"""One repacked device engine per model, shared by every module mirror that wraps the same weights.

The C-ABI engine (``AsrEngine``) repacks a reference-keyed state_dict into an fp16 device arena once.  The nn.Module
mirrors (TransformerASR, the searchers, ConvolutionFrontEnd, EncoderDecoderASR, ...) all want such an engine; building one
each would hold 3-4 copies of the model, and a snapshot taken at first use would silently go stale when
``load_state_dict`` / a checkpoint recovery / ``.to()`` changes the parameters afterwards.  An ``EngineSlot``

* is keyed on the *source modules* (which Linear is the output head, which LM / CTC head the scorers use), so mirrors
  wired to the same modules get the same engine and the union of the parts they need;
* fingerprints every source tensor (``data_ptr``, autograd ``_version``, device): ``load_state_dict`` copies in place and
  bumps ``_version``, ``.to()`` / ``_load`` replace the storage -- either way the next call rebuilds the engine.
  (Edits through ``param.data`` bypass the version counter: call ``invalidate()`` after those.)
"""
import itertools

import torch

_PART_ORDER = ("fbank", "cnn", "encoder", "decoder", "lm")


def _tensors_of(src):
    if isinstance(src, torch.nn.Module):
        extra = [getattr(src, n) for n in ("glob_mean", "glob_std", "_window", "_mel") if torch.is_tensor(getattr(src, n, None))]
        return itertools.chain(src.parameters(), src.buffers(), extra)
    return ()


def fingerprint(sources):
    fp = []
    for name in sorted(sources):
        src = sources[name]
        fp.append((name, id(src)))
        for t in _tensors_of(src):
            fp.append((t.data_ptr(), t._version, str(t.device), tuple(t.shape)))
    return hash(tuple(fp))


class EngineSlot:
    """``cfg_fn() -> dict`` gives the base engine config; ``sources`` maps a weight prefix to the module providing it:
    "Transformer." / "seq_lin." / "ctc_lin." / "CNN." / "lm." (state_dict under that prefix), "normalize"
    (InputNormalization: glob_mean / glob_std / epsilon), "fbank" (Fbank: sizes, window, mel matrix)."""

    def __init__(self, cfg_fn):
        self.cfg_fn = cfg_fn
        self.sources = {}
        self.parts = ()
        self.engine = None
        self._fp = None
        self.builds = 0

    def invalidate(self):
        self.engine = None
        self._fp = None

    def _state_and_cfg(self):
        cfg = dict(self.cfg_fn())
        sd = {}
        for prefix, src in self.sources.items():
            if prefix == "normalize":
                if src.glob_mean.numel() == 0:
                    raise RuntimeError("InputNormalization(global): statistics not loaded (glob_mean is empty)")
                sd["normalize.glob_mean"] = src.glob_mean.detach().float().cpu()
                std = src.glob_std if src.std_norm else torch.ones_like(src.glob_mean)
                sd["normalize.glob_std"] = std.detach().float().cpu()
                cfg["norm_eps"] = float(src.epsilon)
            elif prefix == "fbank":
                cfg.update(n_fft=src.n_fft, hop=src.hop_length, win=src.win_length, n_mels=src.n_mels,
                           sample_rate=src.sample_rate)
                sd["fbank.window"] = src._window.detach().float().cpu()
                sd["fbank.mel_matrix"] = src._mel.detach().float().cpu()
            elif prefix == "lm.":
                sd.update({prefix + k: v for k, v in src.state_dict().items()})
                cfg["lm"] = src.engine_cfg()
            else:
                sd.update({prefix + k: v for k, v in src.state_dict().items()})
                if prefix == "CNN.":
                    cfg["cnn_channels"] = tuple(src.out_channels)
                    cfg["cnn_blocks"] = src.num_blocks  # the front-end actually wired to the model
        return cfg, sd

    def get(self, device, parts, sources=None):
        from .engine import AsrEngine
        device = torch.device(device)
        changed = False
        for prefix, mod in (sources or {}).items():
            if self.sources.get(prefix) is not mod:
                self.sources[prefix] = mod
                changed = True
        want = tuple(p for p in _PART_ORDER if p in set(self.parts) | set(parts))
        fp = fingerprint(self.sources)
        if (self.engine is None or changed or want != self.parts or fp != self._fp or self.engine.device != device):
            cfg, sd = self._state_and_cfg()
            self.engine = None  # free the old arena before allocating the new one
            self.engine = AsrEngine(cfg, sd, device=device, parts=want)
            self.parts, self._fp = want, fp
            self.builds += 1
        return self.engine
