"""Block glue either side of the mixer (SURVEY.md S8 f1): the pre-norm residual Block of the HyenaDNA backbone.

Mirrors flash-attention/flash_attn/modules/block.py:36-200 for the configuration src/models/sequence/long_conv_lm.py
uses (create_block :139-200: prenorm=True, residual_in_fp32, fused_dropout_add_ln optional; LMBackbone.forward :377-396
threads (hidden_states, residual) through the blocks and applies the same dropout -> add -> LayerNorm once more at the
end): same constructor keywords, attribute names (mixer, norm1, mlp, norm2, dropout1/2) and state_dict keys, so a
reference checkpoint's ``backbone.layers.N.*`` entries load unchanged.

The dropout -> add -> LayerNorm step runs as ONE sm_90a kernel (csrc/layernorm.cuh) in fp32 -- the residual stream is
kept in fp32 whatever the activation dtype, i.e. residual_in_fp32 semantics.  Dropout / stochastic depth with p > 0,
post-norm blocks and RMSNorm are outside the hot path and raise; there is no CPU fallback.
"""
import torch
import torch.nn as nn

from . import ops
from ._lib import HyenaB200Error
from .decode import DecodeCache, StepGraph, check_history_dtype


class Block(nn.Module):
    def __init__(self, dim, mixer_cls=None, mlp_cls=None, norm_cls=nn.LayerNorm, dropout_cls=nn.Dropout, prenorm=True,
                 resid_dropout1=0.0, resid_dropout2=0.0, drop_path1=0.0, drop_path2=0.0, fused_dropout_add_ln=False,
                 return_residual=False, residual_in_fp32=False, sequence_parallel=False, mark_shared_params=False):
        super().__init__()
        bad = {"prenorm": not prenorm, "resid_dropout1": resid_dropout1 != 0.0, "resid_dropout2": resid_dropout2 != 0.0,
               "drop_path1": drop_path1 != 0.0, "drop_path2": drop_path2 != 0.0, "return_residual": return_residual,
               "sequence_parallel": sequence_parallel, "mixer_cls": mixer_cls is None}
        bad = [k for k, v in bad.items() if v]
        if bad:
            raise HyenaB200Error(f"Block options outside the sm_90a hot path (no fallback): {bad}")
        self.prenorm = prenorm
        self.fused_dropout_add_ln = fused_dropout_add_ln      # accepted for config compatibility: the fused kernel always runs
        self.return_residual = return_residual
        self.residual_in_fp32 = residual_in_fp32
        self.mixer = mixer_cls(dim)
        self.dropout1 = dropout_cls(resid_dropout1)
        self.norm1 = norm_cls(dim)
        self.mlp = mlp_cls(dim) if mlp_cls is not None else nn.Identity()
        if not isinstance(self.mlp, nn.Identity):
            self.dropout2 = dropout_cls(resid_dropout2)
            self.norm2 = norm_cls(dim)
        for n in (self.norm1, getattr(self, "norm2", None)):
            if n is not None and not isinstance(n, nn.LayerNorm):
                raise HyenaB200Error("Block: only nn.LayerNorm is supported by the fused add + norm kernel")
            if n is not None and not n.elementwise_affine:
                raise HyenaB200Error("Block: the fused add + norm kernel needs an affine LayerNorm (elementwise_affine=True)")
        if mark_shared_params:
            for p in list(self.norm1.parameters()) + (list(self.norm2.parameters()) if hasattr(self, "norm2") else []):
                p._shared_params = True

    @staticmethod
    def _add_norm(hidden_states, residual, norm):
        if not hidden_states.is_cuda:
            raise HyenaB200Error("Block (hyena_b200) runs on CUDA sm_90a only; there is no CPU fallback")
        x = hidden_states.to(torch.float32).contiguous()
        r = residual.to(torch.float32).contiguous() if residual is not None else None
        return ops.add_layer_norm(x, r, norm.weight.to(torch.float32), norm.bias.to(torch.float32) if norm.bias is not None
                                  else None, norm.eps)

    def forward(self, hidden_states, residual=None, mixer_subset=None, mixer_kwargs=None, lengths=None, mask=None):
        """(hidden_states, residual) -> (mlp(LN2(.)) or mixer output, new residual); block.py:111-180, prenorm branch.
        ``lengths``: left-padded rows, passed to the mixer (HyenaOperator.forward); LayerNorm and the MLP act per position.
        ``mask``: the (B, L) attention mask of a left-padded batch, passed to the mixer, differentiable
        (HyenaOperator.forward); with the loss on real positions only, every gradient at the pads is 0."""
        if mixer_subset is not None:
            raise HyenaB200Error("Block: mixer_subset is not supported")
        if mixer_kwargs and mixer_kwargs.get("stream"):
            # streaming forward (HyenaOperator.forward(u, stream=True)): every position of a sequence of any length
            kw = dict(mixer_kwargs)
            self._check_stream(hidden_states, kw.get("inference_params"), lengths, mask, kw.get("cu_seqlens"))
            return self._run_stream(hidden_states, residual, lambda y: self.mixer(y, **kw))
        if mixer_kwargs and mixer_kwargs.get("cu_seqlens") is not None:
            # flash-attention's unpadded convention: hidden_states (total, D), mixer_kwargs cu_seqlens / max_seqlen
            kw = dict(mixer_kwargs)
            kw["cu_seqlens"] = self._check_packed(hidden_states, kw.pop("cu_seqlens"), kw.pop("max_seqlen", None),
                                                  kw.get("inference_params"), lengths, mask)
            return self._run(hidden_states, residual, lambda y: self.mixer(y, **kw))
        if mask is not None:
            kw = dict(mixer_kwargs or {})
            pad = self._check_mask(hidden_states, mask, kw.get("inference_params"), lengths)
            return self._run(hidden_states, residual, lambda y: self.mixer(y, mask=pad, **kw))
        if lengths is not None:
            self._check_lengths(hidden_states, lengths, None, "forward")
            kw = dict(mixer_kwargs or {}, lengths=lengths)
            return self._run(hidden_states, residual, lambda y: self.mixer(y, **kw))
        return self._run(hidden_states, residual, lambda y: self.mixer(y, **(mixer_kwargs or {})))

    def _check_lengths(self, hidden_states, lengths, cache, how):
        if not hasattr(self.mixer, "check_lengths"):
            raise HyenaB200Error(f"Block: the mixer {type(self.mixer).__name__} takes no lengths")
        self.mixer.check_lengths(hidden_states, lengths, cache, how)

    def _check_packed(self, hidden_states, cu_seqlens, max_seqlen=None, cache=None, lengths=None, mask=None):
        if not hasattr(self.mixer, "check_packed"):
            raise HyenaB200Error(f"Block: the mixer {type(self.mixer).__name__} takes no cu_seqlens")
        return self.mixer.check_packed(hidden_states, cu_seqlens, max_seqlen, cache, lengths, mask)

    def _check_packed_decode(self, hidden_states, cache, cu_seqlens, max_seqlen=None, lengths=None, rows=None):
        if not hasattr(self.mixer, "check_packed_decode"):
            raise HyenaB200Error(f"Block: the mixer {type(self.mixer).__name__} takes no packed prompts")
        return self.mixer.check_packed_decode(hidden_states, cache, cu_seqlens, max_seqlen, lengths, rows)

    def _check_stream(self, hidden_states, cache=None, lengths=None, mask=None, cu_seqlens=None, device=True):
        if not hasattr(self.mixer, "check_stream"):
            raise HyenaB200Error(f"Block: the mixer {type(self.mixer).__name__} takes no stream")
        return self.mixer.check_stream(hidden_states, cache, lengths, mask, cu_seqlens, device)

    def _check_mask(self, hidden_states, mask, cache=None, lengths=None):
        if not hasattr(self.mixer, "check_mask"):
            raise HyenaB200Error(f"Block: the mixer {type(self.mixer).__name__} takes no mask")
        return self.mixer.check_mask(hidden_states, mask, cache, lengths)

    def prefill(self, hidden_states, residual, cache, lengths=None, cu_seqlens=None, max_seqlen=None):
        """forward over the first positions, filling the mixer's DecodeCache (HyenaOperator.prefill); ``lengths``:
        left-padded prompts of different lengths; ``cu_seqlens`` / ``max_seqlen``: prompts packed back to back,
        hidden_states (total, D) or (1, total, D)."""
        if cu_seqlens is not None:
            pk = self._check_packed_decode(hidden_states, cache, cu_seqlens, max_seqlen, lengths)[1]
            return self._decode(hidden_states, residual, lambda y: self.mixer.prefill(y, cache, cu_seqlens=pk))
        if lengths is not None:
            self._check_lengths(hidden_states, lengths, cache, "prefill")
            return self._decode(hidden_states, residual, lambda y: self.mixer.prefill(y, cache, lengths))
        return self._decode(hidden_states, residual, lambda y: self.mixer.prefill(y, cache))

    def step(self, hidden_states, residual, cache):
        """forward of one position (B, 1, D) from the mixer's DecodeCache (HyenaOperator.step).  The residual stream of a
        position depends on that position only, so the block keeps no state of its own."""
        return self._decode(hidden_states, residual, lambda y: self.mixer.step(y, cache))

    def extend(self, hidden_states, residual, cache, lengths=None):
        """forward of n more positions (B, n, D) from the mixer's DecodeCache (HyenaOperator.extend); ``lengths`` on a fresh
        cache only (prefill)."""
        if lengths is not None:
            self._check_lengths(hidden_states, lengths, cache, "extend")
            return self._decode(hidden_states, residual, lambda y: self.mixer.extend(y, cache, lengths))
        return self._decode(hidden_states, residual, lambda y: self.mixer.extend(y, cache))

    def admit(self, hidden_states, residual, cache, rows, lengths=None, cu_seqlens=None):
        """forward of k prompts (k, P, D) that join the running cache in the rows ``rows`` (HyenaOperator.admit); the
        outputs are those of ``prefill`` on a fresh k-row cache.  ``cu_seqlens``: the k prompts packed back to back."""
        if not hasattr(self.mixer, "admit"):
            raise HyenaB200Error(f"Block: the mixer {type(self.mixer).__name__} has no incremental decoding")
        if cu_seqlens is not None:
            pk = self._check_packed_decode(hidden_states, cache, cu_seqlens, None, lengths, rows)[1]
            return self._decode(hidden_states, residual, lambda y: self.mixer.admit(y, cache, rows, cu_seqlens=pk))
        self.mixer.check_admit(hidden_states, cache, rows, lengths)
        return self._decode(hidden_states, residual, lambda y: self.mixer.admit(y, cache, rows, lengths))

    def capture_step(self, cache, batch_size=None, dtype=torch.float32, residual=False):
        """A decode.StepGraph of ``step`` on the mixer's cache; ``residual`` says whether steps pass a residual (False for
        a first block)."""
        return StepGraph(self, cache, batch_size, dtype, residual=residual)

    def _decode(self, hidden_states, residual, mix):
        if not hasattr(self.mixer, "step"):
            raise HyenaB200Error(f"Block: the mixer {type(self.mixer).__name__} has no incremental decoding")
        if hidden_states.requires_grad or (residual is not None and residual.requires_grad):
            raise HyenaB200Error("decoding is inference only: the input requires grad (run under torch.no_grad())")
        with torch.no_grad():
            return self._run(hidden_states, residual, mix)

    @staticmethod
    def _stream_add_norm(hidden_states, residual, norm):
        """_add_norm of a (B, L, D) stream in pieces of ops.STREAM_CHUNK_POSITIONS positions of all rows, so that no
        launch takes more positions than a 2^20-position forward: -> (y, residual), both fp32 (B, L, D)."""
        B, L, D = hidden_states.shape
        n = max(1, ops.STREAM_CHUNK_POSITIONS // B)
        y = torch.empty(B, L, D, dtype=torch.float32, device=hidden_states.device)
        res = torch.empty(B, L, D, dtype=torch.float32, device=hidden_states.device)
        for a in range(0, L, n):
            yc, rc = Block._add_norm(hidden_states[:, a:a + n], residual[:, a:a + n] if residual is not None else None,
                                     norm)
            y[:, a:a + n] = yc
            res[:, a:a + n] = rc
        return y, res

    def _run_stream(self, hidden_states, residual, mix):
        """_run for a stream (inference): the mixer runs on the whole sequence (it cuts its own chunks); the fused add +
        LayerNorm and the MLP act per position and run in pieces of ops.STREAM_CHUNK_POSITIONS positions of all rows."""
        in_dtype = hidden_states.dtype
        B, L, _ = hidden_states.shape
        with torch.no_grad():
            y, residual = self._stream_add_norm(hidden_states, residual, self.norm1)
            hidden_states = mix(y.to(in_dtype))
            del y
            if isinstance(hidden_states, tuple):            # mixers built with return_state
                hidden_states = hidden_states[0]
            if not isinstance(self.mlp, nn.Identity):
                y, residual = self._stream_add_norm(hidden_states, residual, self.norm2)
                n = max(1, ops.STREAM_CHUNK_POSITIONS // B)
                out = None
                for a in range(0, L, n):
                    oc = self.mlp(y[:, a:a + n].to(in_dtype))
                    if out is None:
                        out = torch.empty(B, L, oc.shape[-1], dtype=oc.dtype, device=oc.device)
                    out[:, a:a + n] = oc
                hidden_states = out
            if not self.residual_in_fp32:
                residual = residual.to(in_dtype)
        return hidden_states, residual

    def _run(self, hidden_states, residual, mix):
        in_dtype = hidden_states.dtype
        y, residual = self._add_norm(hidden_states, residual, self.norm1)
        hidden_states = mix(y.to(in_dtype))
        if isinstance(hidden_states, tuple):                # mixers built with return_state
            hidden_states = hidden_states[0]
        if not isinstance(self.mlp, nn.Identity):
            y, residual = self._add_norm(hidden_states, residual, self.norm2)
            hidden_states = self.mlp(y.to(in_dtype))
        if not self.residual_in_fp32:
            residual = residual.to(in_dtype)
        return hidden_states, residual


class Backbone(nn.Module):
    """Stack of Blocks + the final dropout -> add -> LayerNorm (LMBackbone without the embedding: long_conv_lm.py:377-396).
    Attribute names follow the reference (``layers``, ``ln_f``) so that its state_dict keys map one to one."""

    def __init__(self, d_model, n_layer, mixer_cls, mlp_cls=None, layer_norm_epsilon=1e-5, residual_in_fp32=False):
        super().__init__()
        self.residual_in_fp32 = residual_in_fp32
        self.layers = nn.ModuleList([
            Block(d_model, mixer_cls=mixer_cls, mlp_cls=mlp_cls, norm_cls=lambda d: nn.LayerNorm(d, eps=layer_norm_epsilon),
                  prenorm=True, residual_in_fp32=residual_in_fp32) for _ in range(n_layer)])
        self.ln_f = nn.LayerNorm(d_model, eps=layer_norm_epsilon)

    def forward(self, hidden_states, lengths=None, mask=None, cu_seqlens=None, max_seqlen=None, stream=False):
        """``lengths``: left-padded rows (HyenaOperator.forward), inference only.  ``mask``: the (B, L) attention mask of a
        left-padded batch (the reference datamodules' ``mask`` batch kwarg), differentiable (HyenaOperator.forward).
        ``cu_seqlens`` / ``max_seqlen``: packed sequences, hidden_states (total, D) or (1, total, D) (HyenaOperator.forward),
        validated once for all layers.  ``stream=True``: every position of a (B, L, D) input of any length, each layer
        streaming its own l_max - 1 positions of context (HyenaOperator.forward(u, stream=True)); inference only, every
        layer checked before the first kernel."""
        if stream:
            for layer in self.layers:
                layer._check_stream(hidden_states, None, lengths, mask, cu_seqlens, device=False)
            self.layers[0]._check_stream(hidden_states)
            residual = None
            for layer in self.layers:
                hidden_states, residual = layer(hidden_states, residual, mixer_kwargs={"stream": True})
            with torch.no_grad():
                y, _ = Block._stream_add_norm(hidden_states, residual, self.ln_f)
                return y.to(hidden_states.dtype)
        if cu_seqlens is not None:
            pk = self.layers[0]._check_packed(hidden_states, cu_seqlens, max_seqlen, None, lengths, mask)
            residual = None
            for layer in self.layers:
                hidden_states, residual = layer(hidden_states, residual, mixer_kwargs={"cu_seqlens": pk})
            y, _ = Block._add_norm(hidden_states, residual, self.ln_f)
            return y.to(hidden_states.dtype)
        if mask is not None:                  # validated once: the layers get the LeftPadding
            mask = self.layers[0]._check_mask(hidden_states, mask, None, lengths)
        if lengths is not None:
            self.layers[0]._check_lengths(hidden_states, lengths, None, "forward")
        residual = None
        for layer in self.layers:
            hidden_states, residual = layer(hidden_states, residual, lengths=lengths, mask=mask)
        y, _ = Block._add_norm(hidden_states, residual, self.ln_f)
        return y.to(hidden_states.dtype)

    def allocate_decode_cache(self, batch_size, max_seqlen, history_dtype=torch.float32):
        """One DecodeCache holding the state of every layer's mixer (decode.py), each history stored as ``history_dtype``.
        ``max_seqlen`` None: unbounded, every layer sliding together (the layers' mixers must share l_max)."""
        check_history_dtype(history_dtype)
        if max_seqlen is None and len({getattr(layer.mixer, "l_max", None) for layer in self.layers}) > 1:
            raise HyenaB200Error("DecodeCache.stack: an unbounded stack needs every layer unbounded with the same l_max")
        return DecodeCache.stack(layer.mixer.allocate_decode_cache(batch_size, max_seqlen, history_dtype)
                                 for layer in self.layers)

    def prefill(self, hidden_states, cache, lengths=None, cu_seqlens=None, max_seqlen=None):
        """forward over the first P positions (B, P, D), filling ``cache`` for step(); ``lengths``: left-padded prompts of
        different lengths; ``cu_seqlens`` / ``max_seqlen``: B prompts packed back to back, hidden_states (total, D) or
        (1, total, D), validated once for all layers (HyenaOperator.prefill)."""
        if cu_seqlens is not None:
            if hidden_states.requires_grad:
                raise HyenaB200Error("decoding is inference only: the input requires grad (run under torch.no_grad())")
            pk = cu_seqlens
            for layer in self.layers:
                pk = layer._check_packed_decode(hidden_states, cache, pk, max_seqlen, lengths)[1]
            return self._packed(hidden_states, lambda layer, h, res: layer.prefill(h, res, cache, cu_seqlens=pk))
        return self._decode(hidden_states, cache, "prefill", lengths)

    def step(self, hidden_states, cache):
        """The output of one more position (B, 1, D)."""
        return self._decode(hidden_states, cache, "step")

    def extend(self, hidden_states, cache, lengths=None):
        """The outputs of n more positions (B, n, D); on a fresh cache this is prefill (``lengths`` there only)."""
        return self._decode(hidden_states, cache, "extend", lengths)

    def admit(self, hidden_states, cache, rows, lengths=None, cu_seqlens=None):
        """k prompts (k, P, D) join the running ``cache`` in the rows ``rows`` (HyenaOperator.admit): the outputs of
        ``prefill`` on a fresh k-row cache.  Every layer is checked, and shifted when P > t, before the first layer admits.
        ``cu_seqlens``: the k prompts packed back to back, hidden_states (total, D) or (1, total, D)."""
        if hidden_states.requires_grad:
            raise HyenaB200Error("decoding is inference only: the input requires grad (run under torch.no_grad())")
        if cu_seqlens is not None:
            pk = cu_seqlens
            for layer in self.layers:
                pk = layer._check_packed_decode(hidden_states, cache, pk, None, lengths, rows)[1]
            with torch.no_grad():
                cache._admit_clock(pk.max_len)
            return self._packed(hidden_states, lambda layer, h, res: layer.admit(h, res, cache, rows, cu_seqlens=pk))
        for layer in self.layers:
            if not hasattr(layer.mixer, "admit"):
                raise HyenaB200Error(f"Block: the mixer {type(layer.mixer).__name__} has no incremental decoding")
            layer.mixer.check_admit(hidden_states, cache, rows, lengths)
        with torch.no_grad():
            cache._admit_clock(hidden_states.shape[1])
            residual = None
            for layer in self.layers:
                hidden_states, residual = layer.admit(hidden_states, residual, cache, rows, lengths)
            y, _ = Block._add_norm(hidden_states, residual, self.ln_f)
            return y.to(hidden_states.dtype)

    def capture_step(self, cache, batch_size=None, dtype=torch.float32):
        """A decode.StepGraph of ``step`` on ``cache``: every layer and ln_f in one CUDA graph per route."""
        return StepGraph(self, cache, batch_size, dtype)

    def _packed(self, hidden_states, run):
        """Packed prompts through every layer (``run(layer, hidden_states, residual)``) and ln_f, under no_grad."""
        with torch.no_grad():
            residual = None
            for layer in self.layers:
                hidden_states, residual = run(layer, hidden_states, residual)
            y, _ = Block._add_norm(hidden_states, residual, self.ln_f)
            return y.to(hidden_states.dtype)

    def _decode(self, hidden_states, cache, how, lengths=None):
        if hidden_states.requires_grad:
            raise HyenaB200Error("decoding is inference only: the input requires grad (run under torch.no_grad())")
        if lengths is not None:
            self.layers[0]._check_lengths(hidden_states, lengths, cache, how)
        elif isinstance(cache, DecodeCache) and cache.unbounded:
            # an unbounded stack is checked before any device work, then slides every layer once, before the first layer
            # runs (each mixer would slide its own cache alike); an extend longer than S runs in pieces inside each mixer,
            # the first being this one
            n = hidden_states.shape[1] if hidden_states.dim() == 3 else -1
            self.layers[0].mixer._decode_checks(hidden_states, cache, n, fresh=how == "prefill")
            if how != "prefill" and cache.t > 0:
                with torch.no_grad():
                    cache._make_room(min(n, cache.slide), step=how == "step")
        with torch.no_grad():
            residual = None
            for layer in self.layers:
                hidden_states, residual = getattr(layer, how)(hidden_states, residual, cache) if lengths is None else \
                    getattr(layer, how)(hidden_states, residual, cache, lengths)
            y, _ = Block._add_norm(hidden_states, residual, self.ln_f)
            return y.to(hidden_states.dtype)
