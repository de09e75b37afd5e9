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

An *unbounded* cache (max_seqlen=None, DESIGN.md section 4.20) has no position limit.  The filter has l_max taps, so the
output at t reads no history position s <= t - l_max: before an operation would pass Lcap, the history slides left past
every position no later output reaches (ops.decode_slide_plan).  Its buffer holds Lcap = unbounded_lcap(l_max) positions
and its stored filter is the l_max taps with zeros up to the row stride, so every kernel runs on it unchanged.
"""
import torch

from ._lib import HyenaB200Error

CHUNK = 1024          # positions per partial dot product of a step (csrc/decode_args.h kChunk)


def _ld(lcap):
    return (lcap + 3) // 4 * 4


def _chunks(lcap):
    return (lcap + CHUNK - 1) // CHUNK


SLIDE_MAX = 4096      # positions an unbounded cache holds beyond its filter's reach (at most)
MAX_LCAP = 1 << 20    # longest history a decode cache can hold (csrc/api.cu check_decode_shape)


def slide_room(l_max):
    """S = min(4096, l_max rounded up to a multiple of 4): the positions an unbounded cache of an operator with l_max filter
    taps has room for after a slide, and the longest piece an extend of it runs at once."""
    return min(SLIDE_MAX, _ld(int(l_max)))


def unbounded_lcap(l_max):
    """Lcap of an unbounded cache: l_max + S + 3 rounded up to a multiple of 4.  A slide leaves t in [l_max - 1, l_max + 2]
    (its shift is rounded down to a multiple of 4), so any n <= S more positions fit after it."""
    return _ld(int(l_max) + slide_room(l_max) + 3)


HISTORY_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def check_history_dtype(history_dtype):
    """The element type of a cache's stored history h (DESIGN.md section 4.16): fp32 (the default), fp16 or bf16."""
    if history_dtype not in HISTORY_DTYPES:
        raise HyenaB200Error(f"history_dtype must be torch.float32, torch.float16 or torch.bfloat16; got {history_dtype!r}")
    return history_dtype


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


def host_lengths(lengths, batch, positions):
    """lengths (a sequence or 1-D tensor of B integers, each in [1, positions]) -> list of ints, checked on the host before
    any device work.  Row b of a left-padded batch holds its real tokens at positions [positions - lengths[b], positions)."""
    if torch.is_tensor(lengths):
        if lengths.dim() != 1 or lengths.dtype.is_floating_point or lengths.dtype.is_complex or lengths.dtype == torch.bool:
            raise HyenaB200Error(f"lengths must be a 1-D integer tensor; got {lengths.dtype} of shape {tuple(lengths.shape)}")
        lengths = lengths.tolist()
    try:
        out = [int(n) for n in lengths]
        if any(isinstance(n, bool) or int(n) != n for n in lengths):
            raise ValueError
    except (TypeError, ValueError):
        raise HyenaB200Error("lengths must be a 1-D sequence of integers") from None
    if len(out) != batch:
        raise HyenaB200Error(f"lengths has {len(out)} entries; the batch has {batch} rows")
    bad = [n for n in out if not 1 <= n <= positions]
    if bad:
        raise HyenaB200Error(f"lengths {bad[0]} outside [1, {positions}] (the padded input has {positions} positions)")
    return out


class _PositionState:
    """The values last written to a device position (None: unknown), shared by every cache that holds the tensor."""

    def __init__(self):
        self.value = None


class DecodeCache:
    """Decoding state of one HyenaOperator (``HyenaOperator.allocate_decode_cache``), or of every mixer of a stack
    (``Backbone.allocate_decode_cache``: ``layers`` holds one per layer, looked up by module identity).

    Per operator, with O = order, D = d_model, F = (O-1) D filter channels, C = (O+1) D in_proj channels and ld = Lcap
    rounded up to a multiple of 4 (all fp32 but h, on the operator's device):
      k     (F * ld + 4,)       the filter, each row time-reversed (k[c][j] at c*ld + ld-1-j) so that the step kernel streams
                                history and filter in ascending order; 4 floats of padding
      bias  (F,)                the effective filter bias (0 * bias when use_bias is false, as in forward)
      h     (O-1, B, D, ld)     g_o of every recurrence by position, in ``history_dtype``: fp32 by default; fp16 or bf16
                                hold g^_o = g_o rounded to nearest even, and every route then computes
                                out_o[t] = sum_{s<=t} k_o[t-s] g^_o[s] + bias_o g^_o[t] in fp32 (DESIGN.md section 4.16)
      tail  (B, C, 2)           in_proj outputs (with bias) of the last two positions
      s_t   (B, C)              short-filter outputs of the current position
      part  (B, D, ceil(Lcap / 1024))  partial dot products of one step
    ``t`` is the number of positions consumed so far.

    Unbounded cache (``allocate(op, B, None)``, DESIGN.md section 4.20): ``reach`` = l_max, the filter's taps, and Lcap =
    unbounded_lcap(l_max); k holds the l_max taps and zeros from tap l_max to ld, so k[j] = 0 for every l_max <= j < ld.
    Every step, extend, StepGraph replay and fork first calls ``_make_room``, which slides every layer left when the next
    positions would pass Lcap (ops.decode_slide_plan, on decode_shift_kernel).  ``dropped`` counts the positions slid out.

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
    operation on a branch reads the context before b.

    Left-padded prefill (``HyenaOperator.prefill(u, cache, lengths)``, DESIGN.md section 4.14): ``start`` is the tuple of the
    rows' first real positions s_b = P - lengths[b] (``start_dev`` the same as a (B,) int32 tensor on the device), None for
    a cache prefilled without lengths.  The history before s_b is zero, exactly the history the unpadded row would have, so
    every later operation runs unchanged; ``lengths`` = t - start is the number of real positions each row holds.  Row b
    can hold at most Lcap - s_b real positions.  ``fork`` gives each branch its parent row's start, ``select`` permutes them.

    Continuous batching (``HyenaOperator.admit``, ``release``, ``compact``; DESIGN.md section 4.15): the rows keep the one
    position t.  A prompt joins a row by being placed so that it ends at t with a zero history before it; ``release`` frees
    a row (``free``, host only) and ``compact`` shifts the history left so that t drops by the smallest live start.  Once a
    cache has been admitted into, ``start`` is defined for every row.

    Device position (``sync_position``, StepGraph): ``pos`` (3,) int32 on the device holds [t, win_b, base] for the step
    kernels that read the position on the device.  One tensor serves every layer of a stack.  It is allocated on first
    use and written only by ``sync_position`` and by a replayed StepGraph; ``t`` on the host stays authoritative."""

    def __init__(self, owner=None, batch_size=0, max_seqlen=0, lcap=0, k=None, bias=None, h=None, tail=None, s_t=None,
                 part=None, layers=None, reach=None):
        self.owner = owner
        self.batch_size, self.lcap = int(batch_size), int(lcap)
        self.max_seqlen = None if max_seqlen is None else int(max_seqlen)
        self.reach, self._dropped = (None if reach is None else int(reach)), 0
        self.k, self.bias, self.h, self.tail, self.s_t, self.part = k, bias, h, tail, s_t, part
        self.layers = list(layers) if layers is not None else []
        self._t = 0
        self.win_b, self.win_wc, self.win_f, self.steps = 0, 0, None, 0
        self._branched, self.base, self.hc, self.f, self.parent = False, 0, 0, None, None
        self.pos, self._pos_state = None, None
        self._start, self.start_dev = None, None
        self._free = frozenset()
        if owner is not None:
            self.d_model, self.order = owner.d_model, owner.order

    @classmethod
    def allocate(cls, op, batch_size, max_seqlen, history_dtype=torch.float32):
        """Decoding state of ``op`` for ``batch_size`` rows and up to min(max_seqlen, op.l_max) positions, with the history
        stored as ``history_dtype`` (torch.float32, torch.float16 or torch.bfloat16).  ``max_seqlen`` None: an unbounded
        cache, which slides past the filter's l_max taps instead of stopping at Lcap (DESIGN.md section 4.20)."""
        check_history_dtype(history_dtype)
        if op.filter_fn.bidirectional:
            raise HyenaB200Error("decoding needs a causal filter; this HyenaFilter is bidirectional")
        lk = cls.check_allocation(batch_size, max_seqlen, op.l_max)
        w = op.in_proj.weight
        if not w.is_cuda:
            raise HyenaB200Error("decoding runs on CUDA sm_90a only; the operator's parameters are on the CPU")
        B, D, O = int(batch_size), op.d_model, op.order
        lcap = unbounded_lcap(lk) if lk is not None else min(int(max_seqlen), op.l_max)
        taps = min(lcap, op.l_max)
        ld = _ld(lcap)
        F = (O - 1) * D
        dev = w.device
        with torch.no_grad():
            k = op.filter_fn.filter_channel_major(taps)                  # (F, taps); zero taps from l_max on
            krev = torch.zeros(F * ld + 4, dtype=torch.float32, device=dev)
            krev[:F * ld].view(F, ld)[:, ld - taps:] = k.flip(-1)
            fb = op.filter_fn.bias if op.filter_fn.use_bias else 0 * op.filter_fn.bias
            fb = fb.detach().reshape(-1).to(torch.float32).contiguous().clone()
        h = torch.zeros(O - 1, B, D, ld, dtype=history_dtype, device=dev)
        tail = torch.zeros(B, (O + 1) * D, 2, dtype=torch.float32, device=dev)
        s_t = torch.zeros(B, (O + 1) * D, dtype=torch.float32, device=dev)
        part = torch.zeros(B, D, _chunks(lcap), dtype=torch.float32, device=dev)
        return cls(op, B, max_seqlen, lcap, krev, fb, h, tail, s_t, part, reach=lk)

    @staticmethod
    def check_allocation(batch_size, max_seqlen, l_max):
        """Host checks of an allocation -> the filter reach l_max of an unbounded cache (``max_seqlen`` None), else None."""
        if max_seqlen is None:
            if batch_size < 1:
                raise HyenaB200Error(f"allocate_decode_cache: batch_size {batch_size} must be >= 1")
            if unbounded_lcap(l_max) > MAX_LCAP:
                raise HyenaB200Error(f"allocate_decode_cache: an unbounded cache holds l_max + S + 3 = "
                                     f"{unbounded_lcap(l_max)} positions (l_max = {l_max}), more than the {MAX_LCAP} a "
                                     "decode cache can hold; give max_seqlen")
            return int(l_max)
        if batch_size < 1 or max_seqlen < 1:
            raise HyenaB200Error(f"allocate_decode_cache: batch_size {batch_size} and max_seqlen {max_seqlen} must be >= 1")
        return None

    @classmethod
    def stack(cls, caches):
        """One cache for several operators (one per layer of a stack), each found by ``for_module``.  The layers of an
        unbounded stack share one filter reach, so that they slide together."""
        caches = list(caches)
        if not caches:
            raise HyenaB200Error("DecodeCache.stack needs at least one operator cache")
        if len({c.reach for c in caches}) > 1:
            raise HyenaB200Error("DecodeCache.stack: an unbounded stack needs every layer unbounded with the same l_max")
        return cls(None, caches[0].batch_size, caches[0].max_seqlen, min(c.lcap for c in caches), layers=caches)

    @staticmethod
    def layout_nbytes(batch_size, d_model, order, lcap, history_dtype=torch.float32):
        """Bytes one operator's cache takes (the layout in the class docstring), its history stored as ``history_dtype``."""
        e = torch.empty(0, dtype=check_history_dtype(history_dtype)).element_size()
        B, D, O = batch_size, d_model, order
        ld, F, C = _ld(lcap), (order - 1) * d_model, (order + 1) * d_model
        return 4 * ((F * ld + 4) + F + B * C * 2 + B * C + B * D * _chunks(lcap)) + e * (O - 1) * B * D * ld

    @property
    def unbounded(self):
        """True for a cache allocated with max_seqlen=None: it slides instead of stopping at Lcap (a branch never is)."""
        return self.layers[0].unbounded if self.layers else self.reach is not None

    @property
    def dropped(self):
        """Positions slid out of an unbounded cache so far, summed over its slides (0 for any other cache): position t of
        the cache is position dropped + t of the sequence, as long as no ``compact`` or right-shifting ``admit`` moved t."""
        return self.layers[0].dropped if self.layers else self._dropped

    @property
    def slide(self):
        """S (``slide_room``) of an unbounded cache, None for any other: the longest piece an extend of it runs at once."""
        if not self.unbounded:
            return None
        return slide_room(self.layers[0].reach if self.layers else self.reach)

    def _make_room(self, n, step=False):
        """Before n more positions of an unbounded cache (``step``: one step, which may open a window): when
        ops.decode_slide_plan asks for it, slide every layer left by m (decode_shift_kernel, one launch per layer) and add m
        to ``dropped``; returns m (0: no slide, or a bounded cache, whose room the callers check)."""
        if not self.unbounded:
            return 0
        from . import ops
        c0 = self.layers[0] if self.layers else self
        shift, _, keep = ops.decode_slide_plan(self.t, n, c0.reach, c0.lcap, *self._window(), step=step)
        if shift == 0:
            return 0
        for c in (self.layers or [self]):
            c._reposition(shift, keep)
            c._dropped -= shift
        return -shift

    @property
    def history_dtype(self):
        """The element type of the stored history h: torch.float32, torch.float16 or torch.bfloat16."""
        return self.layers[0].history_dtype if self.layers else self.h.dtype

    @property
    def nbytes(self):
        """Bytes the cache owns: the layout above, or for a branched cache its branch state (h, f, tail, s_t, part, parent;
        the filter is the parent's)."""
        if self.layers:
            return sum(c.nbytes for c in self.layers)
        own = (self.h, self.f, self.tail, self.s_t, self.part, self.parent) if self.branched else \
              (self.k, self.bias, self.h, self.tail, self.s_t, self.part)
        own += (self.start_dev,) if self.start_dev is not None else ()
        return sum(x.numel() * x.element_size() for x in own)

    @property
    def branched(self):
        return self.layers[0].branched if self.layers else self._branched

    def fork(self, rows, horizon=4096):
        """A branched cache of len(rows) rows: row i continues row ``rows[i]`` of this cache from its current position t0
        (repeat a row for several branches of one context) and can be stepped and extended up to horizon positions past
        its base t0 - t0 mod 4, or to Lcap.  A snapshot: this cache can go on decoding without changing the branches.  A
        stack's cache forks every layer.  An unbounded cache first slides in place when the branches would otherwise get
        fewer than min(horizon, S) positions (DecodeCache._make_room): its outputs do not change, but its t, ``dropped``
        and window move as after any slide."""
        if self.branched:
            raise HyenaB200Error("fork: this cache is branched already; use select() to reorder, repeat or drop branches")
        rows = _host_index(rows, self.batch_size, "fork: rows")
        horizon = int(horizon)
        if horizon < 1:
            raise HyenaB200Error(f"fork: horizon {horizon} must be >= 1")
        if self.unbounded and self.t >= 1:
            self._make_room(min(horizon, self.slide))     # an unbounded parent slides first, so the branches get room
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
        """Close the window and restart the step and slide counts (a prefill starts a new sequence)."""
        self.win_b, self.win_wc, self.steps, self._dropped = 0, 0, 0, 0

    @property
    def start(self):
        """First real position of every row after a left-padded prefill (a tuple), or None; one for all layers of a stack."""
        return self.layers[0].start if self.layers else self._start

    def set_start(self, start):
        """Record the rows' first real positions (None: every row starts at 0), on the host and as (B,) int32 on the device."""
        if self.layers:
            raise HyenaB200Error("the row starts of a stack's cache are set by its layers")
        self._start = None if start is None else tuple(int(s) for s in start)
        self.start_dev = None if start is None else torch.tensor(self._start, dtype=torch.int32, device=self.h.device)

    @property
    def lengths(self):
        """Real positions each row holds: t - start (t for every row of a cache prefilled without lengths), 0 for a row
        released by ``release``."""
        start, free = self.start, self.free
        return tuple(0 if b in free else self.t - (start[b] if start is not None else 0) for b in range(self.batch_size))

    # ------------------------------------------------------------------------ continuous batching (DESIGN.md section 4.15)
    @property
    def free(self):
        """The rows released since they last took a prompt (a frozenset); one set for all layers of a stack."""
        return self.layers[0].free if self.layers else self._free

    def _no_branch(self, what):
        if self.branched:
            raise HyenaB200Error(f"{what}: this cache is branched; admission, release and compaction need a full cache")

    def release(self, rows):
        """Mark ``rows`` free (host only, no device work): they no longer pin compaction, their ``lengths`` read 0, and
        they go on being stepped with the others until ``HyenaOperator.admit`` gives them a new prompt."""
        self._no_branch("release")
        rows = _host_index(rows, self.batch_size, "release: rows")
        for c in (self.layers or [self]):
            c._free = c._free | frozenset(rows)

    def compact(self):
        """Shift the history of every layer left by m, the smallest first real position of a live row rounded down to a
        multiple of 4 (ops.decode_compact_plan), so that t drops by m and every row gains m positions of room; returns m.
        The window is kept when it still holds the position, else closed (the next step refreshes by the usual rule)."""
        self._no_branch("compact")
        from . import ops
        start = self.start if self.start is not None else (0,) * self.batch_size
        shift, _, keep = ops.decode_compact_plan(self.t, start, self.free, *self._window())
        for c in (self.layers or [self]):
            c._reposition(shift, keep)
        return -shift

    def _window(self):
        c = self.layers[0] if self.layers else self
        return c.win_b, c.win_wc

    def _admit_clock(self, P):
        """Make room for prompts of P positions that end at the position (ops.decode_admit_plan), in every layer: at t = 0
        the position moves to P and every row is free until it takes a prompt; when P > t the history shifts right first."""
        from . import ops
        t0 = self.t
        shift, t_new, keep = ops.decode_admit_plan(t0, self.lcap, P, *self._window())
        for c in (self.layers or [self]):
            c._reposition(shift, keep)
            if t0 == 0:
                c._t, c._free = t_new, frozenset(range(c.batch_size))
                c.set_start((t_new,) * c.batch_size)

    def _reposition(self, shift, keep):
        from . import ops
        ops.decode_shift(self, shift)
        if not keep:
            self.win_b, self.win_wc = 0, 0

    def _took(self, rows, starts):
        """Rows ``rows`` of this operator cache took prompts whose first real positions are ``starts``."""
        start = list(self.start) if self.start is not None else [0] * self.batch_size
        for r, s in zip(rows, starts):
            start[r] = s
        self.set_start(start)
        self._free = self._free - frozenset(rows)

    @property
    def t(self):
        return self.layers[0].t if self.layers else self._t

    @t.setter
    def t(self, value):
        if self.layers:
            raise HyenaB200Error("the position of a stack's cache is advanced by its layers")
        self._t = int(value)

    def sync_position(self):
        """The device position ``pos`` = [t, win_b, base] (allocated on first use, one tensor for a stack and all its layers),
        written from the host fields when they differ from the values it was last given."""
        cs = self.layers or [self]
        want = {(c.t, c.win_b, c.base) for c in cs}
        if len(want) != 1:
            raise HyenaB200Error(f"the layers of this stack's cache disagree on (t, win_b, base): {sorted(want)}")
        want = want.pop()
        if self.pos is None or self._pos_state is None:
            pos, state = torch.zeros(3, dtype=torch.int32, device=cs[0].h.device), _PositionState()
            for c in [self] + self.layers:
                c.pos, c._pos_state = pos, state
        if self._pos_state.value != want:
            self.pos.copy_(torch.tensor(want, dtype=torch.int32))
            self._pos_state.value = want
        return self.pos

    def for_module(self, module):
        """The state of ``module`` (this cache itself, or the layer cache allocated for it)."""
        if self.owner is module:
            return self
        for c in self.layers:
            if c.owner is module:
                return c
        raise HyenaB200Error("this DecodeCache was not allocated for this HyenaOperator")


class StepGraph:
    """``step`` of a HyenaOperator, Block or Backbone on one cache, captured in CUDA graphs and replayed per position.

    An eager step costs about 0.1 ms of host and launch time per operator (DESIGN.md section 4.13).  Here the whole step --
    the projections, the step kernels, the add + LayerNorm kernels, the block MLP and ln_f -- is one graph launch.  Its
    kernels read the position from the cache's device position (``DecodeCache.sync_position``), and the last kernel of the
    graph advances it, so every replay steps the next position.  The outputs are the bits eager ``step`` gives on the same
    route.  The routes differ in one case: at t >= WINDOW_MIN_T less than WINDOW_AFTER_STEPS steps after a prefill or an
    extend, eager ``step`` stays on the plain route while a graph step opens a window, whose sums run in another order.

    Routes: the plain step (below ops.WINDOW_MIN_T), the windowed step and the branch step (a branched cache) are separate
    graphs, each captured on first use: warm-up steps on a side stream (their writes to the cache undone), then the capture.
    Before each replay the host runs the route rule on its copy of the position.  When the next position needs a window
    and none holds it, the window is refreshed eagerly, outside the graph, on the current stream: the first step at
    t >= WINDOW_MIN_T opens one, with no run of plain steps before it.  After each replay the host advances ``t`` of every
    layer cache (and the step count of an unbranched one), so eager ``step``, ``extend``, ``fork`` and ``select`` go on
    from there; steps taken eagerly in between are picked up at the next replay.  ``admit``, ``release`` and ``compact``
    between replays write every captured buffer in place and need no recapture; a window they close is reopened at once.

    ``step`` returns static output tensors that the next ``step`` of this object overwrites: copy what you keep.  It
    raises before any device work on an input of another shape, dtype or device than the captured one, at Lcap or a
    branch horizon, and when a buffer the graphs read was replaced since their capture."""

    WARMUP = 2

    def __init__(self, module, cache, batch_size=None, dtype=torch.float32, residual=False):
        from .block import Backbone, Block
        from .hyena import HyenaOperator
        if isinstance(module, HyenaOperator):
            mixers = [module]
        elif isinstance(module, Block):
            mixers = [module.mixer]
        elif isinstance(module, Backbone):
            mixers = [layer.mixer for layer in module.layers]
        else:
            raise HyenaB200Error(f"StepGraph: expected a HyenaOperator, Block or Backbone; got {type(module).__name__}")
        if not all(isinstance(m, HyenaOperator) for m in mixers):
            raise HyenaB200Error("StepGraph: every mixer must be a HyenaOperator (incremental decoding)")
        if not isinstance(cache, DecodeCache):
            raise HyenaB200Error(f"StepGraph needs a DecodeCache, got {type(cache).__name__}")
        if residual and not isinstance(module, Block):
            raise HyenaB200Error("StepGraph: a residual input exists for a Block only")
        self.module, self.mixers = module, mixers
        self.caches = [cache.for_module(m) for m in mixers]
        # the position the graphs advance: the stack's (one for all its layers) or the operator's own
        self.cache = cache if isinstance(module, Backbone) or len(self.caches) > 1 else self.caches[0]
        B = cache.batch_size if batch_size is None else int(batch_size)
        if B != self.caches[0].batch_size:
            raise HyenaB200Error(f"StepGraph: batch size {B} differs from the decode cache's {self.caches[0].batch_size}")
        if any(m.filter_fn.bidirectional for m in mixers):
            raise HyenaB200Error("decoding needs a causal filter; this HyenaFilter is bidirectional")
        self.device = self.caches[0].h.device
        self.shape, self.dtype = (B, 1, mixers[0].d_model), dtype
        self.residual = residual
        self.res_dtype = (torch.float32 if module.residual_in_fp32 else dtype) if residual else None
        self._graphs, self._keys, self._side, self._scratch = {}, {}, None, []
        self._check_room()
        self._slide()
        self._in = torch.zeros(self.shape, dtype=dtype, device=self.device)
        self._res = torch.zeros(self.shape, dtype=self.res_dtype, device=self.device) if residual else None
        self._graph(self.plan()[0])

    # ---------------------------------------------------------------------------------------- host planning
    def plan(self):
        """(route, refresh) of the next step: route "plain", "window" or "branch"; refresh when the window must be opened
        (decode_window_plan with the step count satisfied: a graph step never waits WINDOW_AFTER_STEPS steps)."""
        from . import ops
        c = self.caches[0]
        if c.branched:
            return "branch", False
        route = ops.decode_window_plan(c.t, c.lcap, ops.WINDOW_AFTER_STEPS, c.win_b, c.win_wc)
        return ("window", True) if route == "refresh" else (route, False)

    def _check_room(self):
        c = self.caches[0]
        if c.branched and c.t >= c.base + c.hc:
            raise HyenaB200Error(f"StepGraph: decoding past the branch horizon: position {c.t} is base + Hc = {c.base} + "
                                 f"{c.hc} (fork with a larger horizon, up to Lcap = {c.lcap})")
        if not c.unbounded and c.t >= c.lcap:
            raise HyenaB200Error(f"StepGraph: decoding past the cache: position {c.t} is Lcap = {c.lcap}")

    def _slide(self):
        """An unbounded cache slides eagerly between replays, outside the graphs, once every check has passed
        (DecodeCache._make_room); step() then syncs the position."""
        if self.caches[0].unbounded:
            self.cache._make_room(1, step=True)

    def _check_key(self, route):
        if route in self._keys and self._key(route) != self._keys[route]:
            raise HyenaB200Error("StepGraph.step: a buffer of the decode cache was replaced since the capture (reallocated, "
                                 "re-forked or re-synced elsewhere); capture a new StepGraph")

    _READS = {"plain": ("k", "bias", "h", "tail", "s_t", "part", "pos"),
              "window": ("k", "bias", "h", "tail", "s_t", "part", "pos", "win_f"),
              "branch": ("k", "bias", "h", "tail", "s_t", "part", "pos", "f", "parent")}

    def _key(self, route):
        return tuple((id(x), x.data_ptr()) if x is not None else None
                     for c in self.caches for x in (getattr(c, n) for n in self._READS[route]))

    def _check_input(self, u_t, residual):
        for name, x, dt in (("input", u_t, self.dtype), ("residual", residual, self.res_dtype)):
            if x is None and dt is None:
                continue
            if x is None or dt is None:
                raise HyenaB200Error(f"StepGraph.step: this graph was captured {'with' if dt is not None else 'without'} "
                                     "a residual input")
            if tuple(x.shape) != self.shape or x.dtype != dt or x.device != self.device:
                raise HyenaB200Error(f"StepGraph.step: {name} {tuple(x.shape)} {x.dtype} on {x.device} differs from the "
                                     f"captured {self.shape} {dt} on {self.device}")

    # ---------------------------------------------------------------------------------------- stepping
    def step(self, u_t, residual=None):
        """One position: u_t (B, 1, D) -> the module's step output (a Block's is (hidden_states, residual)), in static
        tensors that the next step overwrites."""
        from . import ops
        self._check_input(u_t, residual)
        self._check_room()
        if self.caches[0].unbounded:
            for r in self._keys:              # any route may run after the slide: all are checked before it
                self._check_key(r)
        self._slide()
        route, refresh = self.plan()
        self._check_key(route)
        if refresh:
            for c in self.caches:
                ops.decode_window_refresh(c)
        graph, out = self._graph(route)
        c0 = self.caches[0]
        t = c0.t
        self.cache.sync_position()
        self._in.copy_(u_t)
        if residual is not None:
            self._res.copy_(residual)
        graph.replay()
        for c in self.caches:
            c.t += 1
            if not c.branched:
                c.steps += 1
        self.cache._pos_state.value = (t + 1, c0.win_b, c0.base)
        return out

    def _graph(self, route):
        """(graph, static output) of ``route``, captured on first use."""
        if route not in self._graphs:
            self._graphs[route] = self._capture(route)
            self._keys[route] = self._key(route)
        return self._graphs[route]

    def _run(self, route):
        """The step on the static inputs with the device-position kernels of ``route``, then the position advance."""
        from . import ops
        from .block import Backbone, Block
        if route == "plain":
            def core(p_t, ib, sw, sb, c):
                return ops.decode_step_dev(p_t, ib, sw, sb, c, min(c.lcap, ops.WINDOW_MIN_T))
        else:
            core = ops.decode_win_step_dev if route == "window" else ops.decode_branch_step_dev

        def mix(op, c):
            return lambda y: op._step_with(y, c, core)
        m = self.module
        with torch.no_grad():
            if isinstance(m, Backbone):
                hidden, res = self._in, None
                for layer, c in zip(m.layers, self.caches):
                    hidden, res = layer._run(hidden, res, mix(layer.mixer, c))
                y, _ = Block._add_norm(hidden, res, m.ln_f)
                out = y.to(hidden.dtype)
            elif isinstance(m, Block):
                out = m._run(self._in, self._res, mix(m.mixer, self.caches[0]))
            else:
                out = m._step_with(self._in, self.caches[0], core)
            ops.decode_pos_advance(self.cache.pos)
        return out

    def _capture(self, route):
        from . import ops
        caches, c0 = self.caches, self.caches[0]
        if route == "window":
            for c in caches:
                if c.win_f is None:           # the refresh writes it in place from now on (decode_window_refresh)
                    c.win_f = torch.zeros(c.order - 1, c.batch_size, c.d_model, ops.WINDOW, dtype=torch.float32,
                                          device=c.h.device)
        pos = self.cache.sync_position()
        # warm-up at the current position: the library's lazy set-up for the capturing stream (cuBLAS workspace, weight
        # images, module loading) happens here, not inside the capture.  A step writes g_t into h and shifts the tail:
        # both are restored.  The warm-up position keeps every route in bounds (window base t - t mod 4).
        j = c0.t - c0.base if c0.branched else c0.t
        saved = [(c.tail.clone(), c.h[..., j].clone()) for c in caches]
        warm = torch.tensor([c0.t, c0.t - c0.t % 4, c0.base], dtype=torch.int32)
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.device)
        side = self._side
        side.wait_stream(torch.cuda.current_stream(self.device))
        # torch's streams are pooled, so the library's per-stream weight-image scratch of the capturing stream could be
        # replaced and freed by other work on it later: the graph gets scratch of its own, held here as long as it lives
        with ops.private_weight_images(self.device, side, self._scratch):
            with torch.cuda.stream(side):
                for _ in range(self.WARMUP):
                    pos.copy_(warm)
                    self._run(route)
                for c, (tail, col) in zip(caches, saved):
                    c.tail.copy_(tail)
                    c.h[..., j].copy_(col)
            torch.cuda.current_stream(self.device).wait_stream(side)
            self.cache._pos_state.value = None
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=side):
                out = self._run(route)
        return graph, out
