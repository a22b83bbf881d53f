"""`Decoder` — drop-in for reference model/decoder.py:9-101.

Same module tree (`layers`, `lout`, `nclass_out`) and PyTorch (out,in) weight layout, so
`load_state_dict(torch.load(...)["geo_decoder"])` (reference shine_batch.py:46-47) and `freeze_model`
(reference utils/tools.py:188-191) work unchanged.  The class-surface methods stay thin torch calls; the hot path
does not come through here but through `fused.sdf_bce_step` / `fused.sdf_infer`, which hand these weights to
the fused sm_90a kernel (`Decoder.c_descriptor`).
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _abi
from .config import SHINEConfig


class Decoder(nn.Module):
    def __init__(self, config: SHINEConfig, is_geo_encoder=True, is_time_conditioned=False):
        super().__init__()
        prefix = "geo" if is_geo_encoder else "sem"
        hidden = getattr(config, f"{prefix}_mlp_hidden_dim")
        bias_on = getattr(config, f"{prefix}_mlp_bias_on")
        depth = getattr(config, f"{prefix}_mlp_level")
        in_dim = config.feature_dim + (1 if is_time_conditioned else 0)
        self.layers = nn.ModuleList(
            [nn.Linear(in_dim if k == 0 else hidden, hidden, bias_on) for k in range(depth)])
        self.lout = nn.Linear(hidden, 1, bias_on)
        self.nclass_out = nn.Linear(hidden, config.sem_class_count + 1, bias_on)  # semantic head (off-path)
        self.to(config.device)

    def _trunk(self, x):
        for layer in self.layers:
            x = F.relu(layer(x))
        return x

    def forward(self, feature):
        return self.sdf(feature)

    def sdf(self, sum_features):
        """Scaled SDF logits, opposite sign to the true SDF (reference model/decoder.py:48-63)."""
        return self.lout(self._trunk(sum_features)).squeeze(1)

    def time_conditionded_sdf(self, sum_features, ts):
        return self.lout(self._trunk(torch.cat((sum_features, ts.view(-1, 1)), dim=1))).squeeze(1)

    def occupancy(self, sum_features):
        return torch.sigmoid(self.sdf(sum_features))

    def sem_label_prob(self, sum_features):
        return F.log_softmax(self.nclass_out(self._trunk(sum_features)), dim=1)

    def sem_label(self, sum_features):
        return torch.argmax(self.sem_label_prob(sum_features), dim=1)

    def __getstate__(self):
        state = self.__dict__.copy()
        state.pop("_desc_cache", None)        # ctypes struct with raw device pointers: never pickled
        return state

    # ---- fused-kernel plumbing ---------------------------------------------------------------------------

    def fused_supported(self) -> bool:
        """The sm_90a fused kernel covers the north-star lattice: F=8 -> 32 -> 32 -> 1."""
        return (len(self.layers) == 2 and self.layers[0].in_features == 8 and self.layers[0].out_features == 32
                and self.layers[1].in_features == 32 and self.layers[1].out_features == 32)

    def fused_params(self):
        """[w1, b1, w2, b2, w3, b3] (bias entries None when geo_mlp_bias_on is False)."""
        l1, l2 = self.layers[0], self.layers[1]
        return [l1.weight, l1.bias, l2.weight, l2.bias, self.lout.weight, self.lout.bias]

    def c_descriptor(self, grads=None) -> _abi.ShineDecoder:
        if not self.fused_supported():
            raise _abi.ShineB200Error(
                "fused sm_90a decoder kernel supports feature_dim=8, geo_mlp_level=2, geo_mlp_hidden_dim=32 only")
        params = self.fused_params()
        sig = (tuple(p.data_ptr() if p is not None else 0 for p in params),
               tuple(g.data_ptr() if g is not None else 0 for g in grads) if grads is not None else None)
        cached = getattr(self, "_desc_cache", None)
        if cached is not None and cached[0] == sig:      # building the ctypes struct costs ~10 us of Python
            return cached[1]
        d = _abi.ShineDecoder()
        names = ("w1", "b1", "w2", "b2", "w3", "b3")
        for name, p in zip(names, params):
            if p is not None:
                _abi.require_cuda(p, "Decoder parameters")
                if not p.is_contiguous() or p.dtype != torch.float32:
                    raise _abi.ShineB200Error("decoder parameters must be contiguous fp32")
                setattr(d, name, p.data_ptr())
        if grads is not None:
            for name, g in zip(names, grads):
                if g is not None:
                    setattr(d, "g" + name, g.data_ptr())
        d.in_dim, d.hidden, d.mlp_level = 8, 32, 2
        object.__setattr__(self, "_desc_cache", (sig, d))
        return d
