"""Incremental decoding state of the causal Hyena operator (the reference leaves HyenaOperator.recurrence unimplemented,
src/models/sequence/hyena.py:384-386, and ignores the ``inference_params`` that LMBackbone threads through,
src/models/sequence/long_conv_lm.py:375-376).

Output t of the causal recurrence o (hyena.py:414-423) is
    out_o[t] = sum_{s<=t} k_o[t-s] g_o[s] + bias_o g_o[t],    g_o = v_o * x_{O-1-o},
so extending a sequence by one position needs the gated inputs g_o of every earlier position, the filter k and the last
two in_proj outputs (the state of the 3-tap short filter) -- not a forward over the whole sequence.  ``DecodeCache`` holds
exactly that; ``HyenaOperator.prefill`` / ``step`` fill and use it (csrc/decode.cuh).

The filter is generated once, at allocation, for Lcap = min(max_seqlen, l_max) positions.  That is valid for any shorter
prefix: k[j] depends on position j only -- z and t are sliced per position, the modulation is per position and the
``normalized`` option divides by the L1 norm over channels at each position (hyena.py:235-236).
"""
import torch

from ._lib import HyenaB200Error

CHUNK = 1024          # positions per partial dot product of a step (csrc/decode_args.h kChunk)


def _ld(lcap):
    return (lcap + 3) // 4 * 4


def _chunks(lcap):
    return (lcap + CHUNK - 1) // CHUNK


def _host_index(index, n, what):
    """index (a sequence or 1-D tensor of integers) -> list of ints in [0, n), checked on the host before any device work."""
    if torch.is_tensor(index):
        if index.dim() != 1 or index.dtype.is_floating_point or index.dtype.is_complex or index.dtype == torch.bool:
            raise HyenaB200Error(f"{what} must be a 1-D integer index; got {index.dtype} of shape {tuple(index.shape)}")
        index = index.tolist()
    try:
        out = [int(i) for i in index]
        if any(isinstance(i, bool) or int(i) != i for i in index):
            raise ValueError
    except (TypeError, ValueError):
        raise HyenaB200Error(f"{what} must be a 1-D sequence of integers") from None
    if not out:
        raise HyenaB200Error(f"{what} is empty")
    bad = [i for i in out if not 0 <= i < n]
    if bad:
        raise HyenaB200Error(f"{what} {bad[0]} outside [0, {n})")
    return out


class DecodeCache:
    """Decoding state of one HyenaOperator (``HyenaOperator.allocate_decode_cache``), or of every mixer of a stack
    (``Backbone.allocate_decode_cache``: ``layers`` holds one per layer, looked up by module identity).

    Per operator, with O = order, D = d_model, F = (O-1) D filter channels, C = (O+1) D in_proj channels and ld = Lcap
    rounded up to a multiple of 4 (all fp32, on the operator's device):
      k     (F * ld + 4,)       the filter, each row time-reversed (k[c][j] at c*ld + ld-1-j) so that the step kernel streams
                                history and filter in ascending order; 4 floats of padding
      bias  (F,)                the effective filter bias (0 * bias when use_bias is false, as in forward)
      h     (O-1, B, D, ld)     g_o of every recurrence by position
      tail  (B, C, 2)           in_proj outputs (with bias) of the last two positions
      s_t   (B, C)              short-filter outputs of the current position
      part  (B, D, ceil(Lcap / 1024))  partial dot products of one step
    ``t`` is the number of positions consumed so far.

    Window state of the windowed step (ops.decode_window_plan, DESIGN.md section 4.11): a window [win_b, win_b + win_wc)
    is valid while win_b <= t < win_b + win_wc; ``win_f`` (O-1, B, D, W) holds F_o[j] = sum_{s < win_b} k_o[win_b+j-s]
    g_o[s] for j < win_wc.  F depends on h[:, :, :, :win_b] only, so an extend inside the window leaves it valid.  It is
    allocated at the first refresh (``window_nbytes``).  ``steps`` counts the steps since the last prefill or extend.

    A *branched* cache (``fork``, ``select``; DESIGN.md section 4.12) holds R branches that continue rows of a parent cache
    from its position t0.  With base b = t0 - t0 mod 4, Hc = min(horizon rounded up to a multiple of 4, Lcap - b) and
    H = Hc rounded up to a multiple of 4, per operator:
      k, bias                the parent's (shared: never written after allocation)
      h     (O-1, R, D, H)   g_o of each branch at positions [b, b + Hc)
      f     (O-1, P, D, H)   F_o[p][j] = sum_{s<b} k_o[b+j-s] g_o[s] of the P distinct forked parent rows, j < Hc
      parent (R,) int32      the row of f each branch reads
      tail, s_t, part        as above with R rows and ceil(H / 1024) partials
    so out_o[t] = F_o[parent][t-b] + sum_{b<=s<t} k_o[t-s] g_o[s] + (k_o[0] + bias_o) g_o[t] for b <= t < b + Hc, and no
    operation on a branch reads the context before b."""

    def __init__(self, owner=None, batch_size=0, max_seqlen=0, lcap=0, k=None, bias=None, h=None, tail=None, s_t=None,
                 part=None, layers=None):
        self.owner = owner
        self.batch_size, self.max_seqlen, self.lcap = int(batch_size), int(max_seqlen), int(lcap)
        self.k, self.bias, self.h, self.tail, self.s_t, self.part = k, bias, h, tail, s_t, part
        self.layers = list(layers) if layers is not None else []
        self._t = 0
        self.win_b, self.win_wc, self.win_f, self.steps = 0, 0, None, 0
        self._branched, self.base, self.hc, self.f, self.parent = False, 0, 0, None, None
        if owner is not None:
            self.d_model, self.order = owner.d_model, owner.order

    @classmethod
    def allocate(cls, op, batch_size, max_seqlen):
        """Decoding state of ``op`` for ``batch_size`` rows and up to min(max_seqlen, op.l_max) positions."""
        if op.filter_fn.bidirectional:
            raise HyenaB200Error("decoding needs a causal filter; this HyenaFilter is bidirectional")
        if batch_size < 1 or max_seqlen < 1:
            raise HyenaB200Error(f"allocate_decode_cache: batch_size {batch_size} and max_seqlen {max_seqlen} must be >= 1")
        w = op.in_proj.weight
        if not w.is_cuda:
            raise HyenaB200Error("decoding runs on CUDA sm_90a only; the operator's parameters are on the CPU")
        B, D, O = int(batch_size), op.d_model, op.order
        lcap = min(int(max_seqlen), op.l_max)
        ld = _ld(lcap)
        F = (O - 1) * D
        dev = w.device
        with torch.no_grad():
            k = op.filter_fn.filter_channel_major(lcap)                  # (F, lcap)
            krev = torch.zeros(F * ld + 4, dtype=torch.float32, device=dev)
            krev[:F * ld].view(F, ld)[:, ld - lcap:] = k.flip(-1)
            fb = op.filter_fn.bias if op.filter_fn.use_bias else 0 * op.filter_fn.bias
            fb = fb.detach().reshape(-1).to(torch.float32).contiguous().clone()
        h = torch.zeros(O - 1, B, D, ld, dtype=torch.float32, device=dev)
        tail = torch.zeros(B, (O + 1) * D, 2, dtype=torch.float32, device=dev)
        s_t = torch.zeros(B, (O + 1) * D, dtype=torch.float32, device=dev)
        part = torch.zeros(B, D, _chunks(lcap), dtype=torch.float32, device=dev)
        return cls(op, B, max_seqlen, lcap, krev, fb, h, tail, s_t, part)

    @classmethod
    def stack(cls, caches):
        """One cache for several operators (one per layer of a stack), each found by ``for_module``."""
        caches = list(caches)
        if not caches:
            raise HyenaB200Error("DecodeCache.stack needs at least one operator cache")
        return cls(None, caches[0].batch_size, caches[0].max_seqlen, min(c.lcap for c in caches), layers=caches)

    @staticmethod
    def layout_nbytes(batch_size, d_model, order, lcap):
        """Bytes one operator's cache takes (the layout in the class docstring)."""
        B, D, O = batch_size, d_model, order
        ld, F, C = _ld(lcap), (order - 1) * d_model, (order + 1) * d_model
        return 4 * ((F * ld + 4) + F + (O - 1) * B * D * ld + B * C * 2 + B * C + B * D * _chunks(lcap))

    @property
    def nbytes(self):
        """Bytes the cache owns: the layout above, or for a branched cache its branch state (h, f, tail, s_t, part, parent;
        the filter is the parent's)."""
        if self.layers:
            return sum(c.nbytes for c in self.layers)
        own = (self.h, self.f, self.tail, self.s_t, self.part, self.parent) if self.branched else \
              (self.k, self.bias, self.h, self.tail, self.s_t, self.part)
        return sum(x.numel() * x.element_size() for x in own)

    @property
    def branched(self):
        return self.layers[0].branched if self.layers else self._branched

    def fork(self, rows, horizon=4096):
        """A branched cache of len(rows) rows: row i continues row ``rows[i]`` of this cache from its current position t0
        (repeat a row for several branches of one context) and can be stepped and extended up to horizon positions past
        its base t0 - t0 mod 4, or to Lcap.  A snapshot: this cache can go on decoding without changing the branches.  A
        stack's cache forks every layer."""
        if self.branched:
            raise HyenaB200Error("fork: this cache is branched already; use select() to reorder, repeat or drop branches")
        rows = _host_index(rows, self.batch_size, "fork: rows")
        horizon = int(horizon)
        if horizon < 1:
            raise HyenaB200Error(f"fork: horizon {horizon} must be >= 1")
        for c in (self.layers or [self]):
            if c.owner.filter_fn.bidirectional:
                raise HyenaB200Error("decoding needs a causal filter; this HyenaFilter is bidirectional")
            if c.t < 1 or c.t >= c.lcap:
                raise HyenaB200Error(f"fork: the cache is at position {c.t}; forking needs 1 <= t0 < Lcap = {c.lcap}")
        from . import ops
        if self.layers:
            return DecodeCache.stack(ops.decode_fork(c, rows, horizon) for c in self.layers)
        return ops.decode_fork(self, rows, horizon)

    def select(self, index):
        """A branched cache of the branches ``index`` of this one (repeats allowed): each row copies that branch's history,
        tail and parent row; F is shared.  Reorders, prunes or re-forks beams in one call."""
        if not self.branched:
            raise HyenaB200Error("select: this cache is not branched (fork() first)")
        index = _host_index(index, self.batch_size, "select: index")
        from . import ops
        if self.layers:
            return DecodeCache.stack(ops.decode_select(c, index) for c in self.layers)
        return ops.decode_select(self, index)

    @property
    def window_nbytes(self):
        """Bytes of the windowed step's history tails (0 until the first window opens); not part of ``nbytes``."""
        if self.layers:
            return sum(c.window_nbytes for c in self.layers)
        return 0 if self.win_f is None else self.win_f.numel() * self.win_f.element_size()

    def reset_window(self):
        """Close the window and restart the step count (a prefill starts a new sequence)."""
        self.win_b, self.win_wc, self.steps = 0, 0, 0

    @property
    def t(self):
        return self.layers[0].t if self.layers else self._t

    @t.setter
    def t(self, value):
        if self.layers:
            raise HyenaB200Error("the position of a stack's cache is advanced by its layers")
        self._t = int(value)

    def for_module(self, module):
        """The state of ``module`` (this cache itself, or the layer cache allocated for it)."""
        if self.owner is module:
            return self
        for c in self.layers:
            if c.owner is module:
                return c
        raise HyenaB200Error("this DecodeCache was not allocated for this HyenaOperator")
