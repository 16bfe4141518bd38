"""Continuous batching: generation requests enter and leave a running batch at step boundaries.

`LMModel.generate` decodes one batch from start to end: every row shares one device position, one text length and one
length, so a service with requests of different durations arriving at different times either runs small batches or runs
each group to its longest member.  A `SlotSession` instead keeps `slots` independent requests on the device
(acb_lm_begin_slots): each slot has its own position, text length, sequence length and seed, a request is admitted into a
free slot between steps and retires when its last column is sampled, while the other slots keep decoding.  The GEMMs still
read every weight byte once per step for all rows.

A request in a session computes what `LMModel.generate` computes for it alone: the same delay-pattern sequence, its own
condition (no padding to other requests' text lengths), and Philox noise keyed by its own seed and column.  Its tokens are
bit-identical to `generate` of that item alone when both run the same GEMM regime (up to 64 rows, i.e. <= 32 slots) and the
prompt is not prefilled (``ACB_LM_PREFILL=0``): a session consumes a continuation prompt one column per step (teacher
forcing), which costs one step per prompt column, where `generate` prefills it several positions per pass.  A request with
`prefill_cols` (`ContinuousGenerator(prefill_prompts=True)`) has its prompt prefilled at admission in `generate`'s passes
(acb_lm_admit_prompt) and equals `generate`'s default path; such a session also runs requests longer than max_duration
window by window (`WindowChain`), re-admitting each window into its slot as the previous one finishes.

A melody model (the `prepend` fuser: MusicGen-melody) conditions a request on a prefix [2, P, d] of chroma and, in the
released layout, description positions, whose length P differs from request to request.  Admission prefills it into the
slot's own cache rows (acb_lm_admit_prefix), in the passes `generate` runs for that request alone, and the slot then runs
column t at cache position P + t.  A session is sized for `max_prefix` prefix positions.

With a KV budget (`SlotSession(kv_pages=N)`, `continuous(kv_cache_gb=...)`) the session's self-attention cache is a pool of
pages of ACB_LM_KV_PAGE positions (acb_lm_begin_slots_paged) instead of `slots` rows of the longest length: a request holds
2 * ceil((P + S) / ACB_LM_KV_PAGE) pages (its cond and null rows) from admission until it finishes or is cancelled, so
the number of requests decoding at once follows their lengths.  A request computes exactly what it computes in a
contiguous session; only the addresses of its keys and values differ.

Each request has its own sampling options (use_sampling, temperature, top-k, top-p, CFG coefficient): admission writes them to
the slot's record on the device, which the captured step reads, so requests with different options share one session.  A
request can be cancelled between steps (acb_lm_retire), which frees its slot for the next admission.

`ContinuousScheduler` is the host-side policy (FIFO admission, head-of-line waiting for pages, retirement, cancellation)
over any object with the device
session's methods, so it is tested without a GPU.  `CohortStream` turns a session's progress into audio pieces while the
requests decode; `ContinuousGenerator` (``BaseGenModel.continuous``) is the public entry point.
"""
import collections
import ctypes as C
import itertools
import math
import typing as tp
from dataclasses import dataclass, field

import torch

from . import _lib
from .musicgen import window_plan

SLOT_INACTIVE, SLOT_ACTIVE, SLOT_FINISHED = 0, 1, 2


@dataclass
class Request:
    """One generation request at the LM level: cross [2, T, d] ([cond; null]) or None, prompt codes [1, K, T0] or None, and
    on a model with a condition prefix its prefix [2, P, d] ([cond; null])."""
    max_gen_len: int
    cross: tp.Optional[torch.Tensor] = None
    prompt: tp.Optional[torch.Tensor] = None
    seed: int = 0
    id: int = -1
    meta: tp.Dict[str, tp.Any] = field(default_factory=dict)   # filled by the session at admission
    # the request's own sampling options; None takes the session's (SlotSession's constructor arguments)
    use_sampling: tp.Optional[bool] = None
    temp: tp.Optional[float] = None
    top_k: tp.Optional[int] = None
    top_p: tp.Optional[float] = None
    cfg_coef: tp.Optional[float] = None
    prefix: tp.Optional[torch.Tensor] = None
    # prompt columns prefilled at admission (acb_lm_admit_prompt); the slot starts decoding at this column
    prefill_cols: int = 0
    # a request longer than the session's max_duration: the windows after this one (None: this is the whole request)
    chain: tp.Optional['WindowChain'] = None


SAMPLING_OPTIONS = ('use_sampling', 'temp', 'top_k', 'top_p', 'cfg_coef')


def check_sampling(use_sampling, temp, top_k, top_p, cfg_coef):
    """The options acb_lm_admit accepts: temp >= 0, an integer top_k >= 0, 0 <= top_p <= 1 and a finite cfg_coef."""
    if not isinstance(use_sampling, (bool, int)):
        raise ValueError(f"use_sampling must be a bool, got {use_sampling!r}")
    if not (isinstance(temp, (int, float)) and math.isfinite(temp) and temp >= 0):
        raise ValueError(f"temperature must be finite and >= 0, got {temp!r}")
    if isinstance(top_k, bool) or not isinstance(top_k, int) or top_k < 0:
        raise ValueError(f"top_k must be an integer >= 0, got {top_k!r}")
    if not (isinstance(top_p, (int, float)) and 0 <= top_p <= 1):
        raise ValueError(f"top_p must be in [0, 1], got {top_p!r}")
    if not (isinstance(cfg_coef, (int, float)) and math.isfinite(cfg_coef)):
        raise ValueError(f"cfg_coef must be finite, got {cfg_coef!r}")


def prefix_bound(lm, max_text: int) -> int:
    """The longest condition prefix a request can have on `lm`: 0 without a `prepend` fuser, else the melody conditioner's
    chroma_len, plus max_text when the description is prepended too (the released [self_wav, description] layout)."""
    if not lm.has_prefix:
        return 0
    cp = getattr(lm, 'condition_provider', None)
    chroma = cp.conditioners['self_wav'] if cp is not None and 'self_wav' in cp.conditioners else None
    if chroma is None or not chroma.match_len_on_eval:
        raise NotImplementedError("a condition prefix without a melody ('self_wav') conditioner matched to its training length "
                                  "has no length bound: pass max_prefix")
    return chroma.chroma_len + (max_text if 'description' in lm.fuser.fuse2cond.get('prepend', []) else 0)


KV_DTYPES = ('fp16', 'fp8')


def check_kv_dtype(kv_dtype) -> str:
    if kv_dtype not in KV_DTYPES:
        raise ValueError(f"the KV cache dtype must be one of {KV_DTYPES}, got {kv_dtype!r}")
    return kv_dtype


def kv_page_bytes(lm, kv_dtype: str = 'fp16') -> int:
    """Bytes of one page of a paged session's pool: ACB_LM_KV_PAGE positions of K and V in every layer, fp16
    (64 L 4 d) or 'fp8': e4m3 codes and one fp32 scale per position and head (64 L (2 d + 8 H))."""
    page, L, d = _lib.ACB_LM_KV_PAGE, lm.num_layers, lm.dim
    if check_kv_dtype(kv_dtype) == 'fp8':
        return page * L * (2 * d + 8 * lm.num_heads)
    return page * 2 * L * d * 2


def kv_pages_for_budget(lm, kv_cache_gb: float, kv_dtype: str = 'fp16') -> int:
    """The pages a budget of kv_cache_gb * 1e9 bytes holds: floor(kv_cache_gb * 1e9 / kv_page_bytes(lm, kv_dtype))."""
    if isinstance(kv_cache_gb, bool) or not isinstance(kv_cache_gb, (int, float)) or not (
            math.isfinite(kv_cache_gb) and kv_cache_gb > 0):
        raise ValueError(f"kv_cache_gb must be a finite number > 0, got {kv_cache_gb!r}")
    return int(math.floor(kv_cache_gb * 1e9 / kv_page_bytes(lm, kv_dtype)))


class PagePool:
    """Host bookkeeping of a paged session's KV pages: the free page ids and the pages each live slot holds.  A request of
    `positions` = P + S cache positions takes `need(positions)` = 2 * ceil(positions / ACB_LM_KV_PAGE) pages, its cond row's
    then its null row's."""

    def __init__(self, n_pages: int):
        self.n_pages = n_pages
        self.free = list(range(n_pages - 1, -1, -1))   # pop() hands out the lowest ids first
        self.held: tp.Dict[int, tp.List[int]] = {}
        self.peak = 0

    @staticmethod
    def need(positions: int) -> int:
        return 2 * -(-positions // _lib.ACB_LM_KV_PAGE)

    def fits(self, positions: int) -> bool:
        return self.need(positions) <= len(self.free)

    @property
    def in_use(self) -> int:
        return self.n_pages - len(self.free)

    def take(self, slot: int, positions: int) -> tp.List[int]:
        if slot in self.held:
            raise RuntimeError(f"slot {slot} still holds pages")
        n = self.need(positions)
        if n > len(self.free):
            raise RuntimeError(f"{positions} positions need {n} pages; {len(self.free)} are free")
        ids = [self.free.pop() for _ in range(n)]
        self.held[slot] = ids
        self.peak = max(self.peak, self.in_use)
        return ids

    def release(self, slot: int):
        self.free.extend(reversed(self.held.pop(slot, [])))


def pattern_sequence(lm, prompt: tp.Optional[torch.Tensor], max_gen_len: int, device='cpu'):
    """The delay-pattern sequence [1, K, S] and mask [K, S] `LMModel._generate_begin` builds for one item: the prompt written
    in, -1 where a token is still unknown, the special token where the pattern has no step.  Also returns the pattern."""
    K = lm.n_q
    if prompt is None:
        prompt = torch.zeros((1, K, 0), dtype=torch.long, device=device)
    prompt = prompt.to(device, torch.long)
    assert prompt.shape[:2] == (1, K), "Inconsistent inputs shapes"
    assert prompt.shape[-1] < max_gen_len
    pattern = lm.pattern_provider.get_pattern(max_gen_len)
    gen_codes = torch.full((1, K, max_gen_len), -1, dtype=torch.long, device=device)
    gen_codes[..., :prompt.shape[-1]] = prompt
    gen_sequence, _, mask = pattern.build_pattern_sequence(gen_codes, lm.special_token_id)
    return gen_sequence, mask, pattern


def prefill_columns(lm, prompt_len: int, max_gen_len: int) -> int:
    """The prompt columns `LMModel.generate` prefills for a prompt of `prompt_len` frames in a generation of max_gen_len
    (`lm.prompt_prefill_columns`): 0 below the pass threshold or with ACB_LM_PREFILL=0."""
    from .lm import prompt_prefill_columns
    return prompt_prefill_columns(lm.pattern_provider.get_pattern(max_gen_len).get_first_step_with_timesteps(prompt_len))


class WindowChain:
    """The windows of one request longer than the session's max_duration, as `BaseGenModel._token_windows` runs them
    (`musicgen.window_plan`).  `make(k, prompt)` builds window k's Request from its prompt; `advance(codes)` takes a finished
    window's codes [1, K, length] and returns the next window's Request (prompted with codes[:, :, stride:]) or None after
    the last.  `tokens()` is then the request's result: its prompt, then each window's new frames."""

    def __init__(self, plan, make: tp.Callable[[int, tp.Optional[torch.Tensor]], Request],
                 prompt: tp.Optional[torch.Tensor]):
        self.plan, self.make, self.k = plan, make, 0
        self.pieces: tp.List[torch.Tensor] = [] if prompt is None else [prompt]

    def advance(self, codes: torch.Tensor) -> tp.Optional[Request]:
        w = self.plan[self.k]
        self.pieces.append(codes[:, :, w.prompt_len:])
        self.k += 1
        return self.make(self.k, codes[:, :, w.stride:]) if self.k < len(self.plan) else None

    def tokens(self) -> torch.Tensor:
        return torch.cat(self.pieces, dim=-1)


def revert_sequence(lm, gen_sequence: torch.Tensor, mask: torch.Tensor, pattern, max_gen_len: int) -> torch.Tensor:
    """`LMModel._generate_end` for one finished item: the checks of lm.py:568-586, then revert_pattern_sequence -> [1, K, T]."""
    unknown_token = -1
    assert not (gen_sequence == unknown_token).any()
    assert (gen_sequence == torch.where(mask[None, ...].expand(gen_sequence.shape[0], -1, -1), gen_sequence,
                                        lm.special_token_id)).all()
    out_codes, _, out_mask = pattern.revert_pattern_sequence(gen_sequence, special_token=unknown_token)
    assert (out_codes[..., :max_gen_len] != unknown_token).all()
    assert (out_mask[..., :max_gen_len] == 1).all()
    out_codes = out_codes[..., :max_gen_len]
    assert (out_codes >= 0).all() and (out_codes <= lm.card).all()
    return out_codes


class SlotSession:
    """The device half of continuous batching on one `LMModel`: `slots` requests decoded side by side, in the CFG layout
    (slot s owns rows s and slots + s).  Holds the model's decode handle until another generation call takes it.

    On a model with a condition prefix every request carries one of at most `max_prefix` positions (None: `prefix_bound`),
    and the KV cache holds max_prefix + the longest sequence.

    `kv_pages`: a paged session.  Its self-attention cache is a pool of `kv_pages` pages (`kv_page_bytes` each) instead of
    2 * slots rows of max_prefix + the longest sequence, and `pages` (a `PagePool`) tracks which slot holds which pages:
    admission takes a request's pages, `collect` and `retire` return them.  Refused (ValueError, before any device work)
    when the pool cannot hold one request of the longest sequence with max_prefix.  Besides the pool the session allocates
    the cross-attention K/V for 2 * slots x max_text positions, a staging cache of 2 x max_prefix positions for admitting a
    prefix, and the activation and split-K buffers of 2 * slots rows.

    `kv_dtype='fp8'` (paged sessions only; ValueError otherwise, before any device work): the pool holds each K or V vector
    of 64 values as e4m3 codes (`k_pool` / `v_pool`, torch.float8_e4m3fn) and one fp32 scale (`k_scale` / `v_scale`
    [L, kv_pages, H, ACB_LM_KV_PAGE]), acb_lm_begin_slots_paged_fp8.  Quantization is local to one row and position, so a
    request's result is that of the same request alone in an fp8 session, but no longer that of an fp16 session."""

    def __init__(self, lm, slots: int, max_gen_len: int, max_text: int = 64, use_sampling: bool = True, temp: float = 1.0,
                 top_k: int = 250, top_p: float = 0.0, cfg_coef: tp.Optional[float] = None,
                 max_prefix: tp.Optional[int] = None, kv_pages: tp.Optional[int] = None, kv_dtype: str = 'fp16'):
        if not 1 <= slots <= _lib.ACB_LM_MAX_SLOTS:
            raise ValueError(f"slots must be in [1, {_lib.ACB_LM_MAX_SLOTS}], got {slots}")
        self.kv_dtype = check_kv_dtype(kv_dtype)
        if kv_dtype == 'fp8' and kv_pages is None:
            raise ValueError("kv_dtype='fp8' is built for paged sessions only: pass kv_pages")
        if max_gen_len < 1 or max_text < 1:
            raise ValueError("max_gen_len and max_text must be >= 1")
        if not lm.has_prefix and max_prefix:
            raise ValueError("max_prefix > 0 needs a model with a condition prefix (prepend fuser)")
        max_prefix = prefix_bound(lm, max_text) if max_prefix is None else int(max_prefix)
        if max_prefix < 0:
            raise ValueError(f"max_prefix must be >= 0, got {max_prefix}")
        self.lm, self.slots, self.max_gen_len, self.max_text = lm, slots, max_gen_len, max_text
        self.max_prefix = max_prefix
        seq, _, pattern = pattern_sequence(lm, None, max_gen_len)
        self.seq_len_max, self.delays = seq.shape[-1], list(pattern.delays)
        self._seq_lens = {max_gen_len: self.seq_len_max}
        coef = lm.cfg_coef if cfg_coef is None else cfg_coef
        self.sampling = dict(use_sampling=bool(use_sampling), temp=float(temp), top_k=int(top_k), top_p=float(top_p),
                             cfg_coef=float(coef))
        self.pages = None
        if kv_pages is not None:
            if isinstance(kv_pages, bool) or not isinstance(kv_pages, int):
                raise ValueError(f"kv_pages must be an integer, got {kv_pages!r}")
            longest = max_prefix + self.seq_len_max
            if kv_pages < PagePool.need(longest):
                raise ValueError(f"a pool of {kv_pages} KV pages cannot hold one request of {longest} positions "
                                 f"({PagePool.need(longest)} pages of {_lib.ACB_LM_KV_PAGE} positions, cond and null rows)")
            self.pages = PagePool(kv_pages)
        with torch.cuda.device(lm.device):
            sizes = (2 * slots, max_prefix + self.seq_len_max, max_text if lm.cross_attention else 0, slots)
            if self.pages is None:
                lm._ensure(*sizes)
            else:
                lm._ensure(*sizes, paged=True)
            samp = _lib.LMSampling(int(bool(use_sampling)), float(temp), int(top_k), float(top_p), float(coef), 0, 0, 0.0)
            if self.pages is None:
                _lib.check(lm._lib.acb_lm_begin_slots(lm._handle, slots, max_text, self.seq_len_max, C.byref(samp),
                                                      _lib.stream()), 'lm_begin_slots')
            else:
                L, H, page, f16 = lm.num_layers, lm.num_heads, _lib.ACB_LM_KV_PAGE, torch.float16
                per_row = PagePool.need(max_prefix + self.seq_len_max) // 2
                # never read before written: a slot reads only the positions it has appended or had scattered in
                code = torch.float8_e4m3fn if kv_dtype == 'fp8' else f16
                self.k_pool = torch.empty((L, kv_pages, H, page, 64), device=lm.device, dtype=code)
                self.v_pool = torch.empty((L, kv_pages, H, page, 64), device=lm.device, dtype=code)
                self.page_table = torch.zeros((2 * slots, per_row), device=lm.device, dtype=torch.int32)
                self._stage = [torch.empty((L, 2, H, max_prefix, 64), device=lm.device, dtype=f16) if max_prefix else None
                               for _ in range(2)]
                if kv_dtype == 'fp8':
                    self.k_scale = torch.empty((L, kv_pages, H, page), device=lm.device, dtype=torch.float32)
                    self.v_scale = torch.empty((L, kv_pages, H, page), device=lm.device, dtype=torch.float32)
                    _lib.check(lm._lib.acb_lm_begin_slots_paged_fp8(
                        lm._handle, slots, max_text, self.seq_len_max, max_prefix, _lib.ptr(self.k_pool),
                        _lib.ptr(self.v_pool), _lib.ptr(self.k_scale), _lib.ptr(self.v_scale), kv_pages,
                        _lib.ptr(self.page_table), per_row, _lib.ptr(self._stage[0]), _lib.ptr(self._stage[1]),
                        C.byref(samp), _lib.stream()), 'lm_begin_slots_paged_fp8')
                else:
                    _lib.check(lm._lib.acb_lm_begin_slots_paged(
                        lm._handle, slots, max_text, self.seq_len_max, max_prefix, _lib.ptr(self.k_pool),
                        _lib.ptr(self.v_pool), kv_pages, _lib.ptr(self.page_table), per_row, _lib.ptr(self._stage[0]),
                        _lib.ptr(self._stage[1]), C.byref(samp), _lib.stream()), 'lm_begin_slots_paged')
            lm.launches_per_step = lm._lib.acb_lm_launches_per_step(lm._handle)
            lm._session = self
            self._status = torch.zeros((slots, 2), device=lm.device, dtype=torch.int32)

    def _check_owner(self):
        if self.lm._session is not self:
            raise RuntimeError("the LM's decode handle was taken by another generation call; start a new session")

    @property
    def max_delay(self) -> int:
        return max(self.delays)

    def positions(self, req: Request) -> int:
        """Cache positions the request occupies in each of its two rows: its prefix and its delay-pattern sequence."""
        n = req.max_gen_len
        if n not in self._seq_lens:
            self._seq_lens[n] = pattern_sequence(self.lm, None, n)[0].shape[-1]
        return (0 if req.prefix is None else req.prefix.shape[1]) + self._seq_lens[n]

    def admit(self, slot: int, req: Request):
        """Write the request's sequence and mask rows, then its sampling options, cross K/V, condition prefix and slot state
        (acb_lm_admit_prefix), and with req.prefill_cols > 0 prefill that many prompt columns (acb_lm_admit_prompt)."""
        self._check_owner()
        lm = self.lm
        if req.max_gen_len > self.max_gen_len:
            raise ValueError(f"max_gen_len {req.max_gen_len} > the session's {self.max_gen_len}")
        samp = None
        if any(getattr(req, k) is not None for k in SAMPLING_OPTIONS):
            o = {k: self.sampling[k] if getattr(req, k) is None else getattr(req, k) for k in SAMPLING_OPTIONS}
            check_sampling(**o)
            samp = C.byref(_lib.LMSampling(int(bool(o['use_sampling'])), float(o['temp']), int(o['top_k']), float(o['top_p']),
                                           float(o['cfg_coef']), 0, 0, 0.0))
        if lm.has_prefix and req.prefix is None:
            raise ValueError("the model prepends a condition prefix: the request needs its prefix [2, P, d]")
        if not lm.has_prefix and req.prefix is not None:
            raise ValueError("the model has no condition prefix (prepend fuser): the request must not carry one")
        P = 0
        if req.prefix is not None:
            if req.prefix.dim() != 3 or req.prefix.shape[0] != 2 or req.prefix.shape[2] != lm.dim:
                raise ValueError(f"prefix must be [2, P, {lm.dim}] ([cond; null]), got {tuple(req.prefix.shape)}")
            P = req.prefix.shape[1]
            if P > self.max_prefix:
                raise ValueError(f"condition prefix of {P} positions: the session holds 0 .. {self.max_prefix}")
        with torch.cuda.device(lm.device):
            seq, mask, pattern = pattern_sequence(lm, req.prompt, req.max_gen_len, lm.device)
            S = seq.shape[-1]
            if not 0 <= req.prefill_cols <= S - 2:
                raise ValueError(f"prefill_cols {req.prefill_cols} not in [0, {S - 2}]")
            b = lm._bufs
            b['seq'][slot].fill_(-1)
            b['seq'][slot, :, :S] = seq[0]
            b['slot_mask'][slot].zero_()
            b['slot_mask'][slot, :, :S] = mask.to(torch.uint8)
            cross, T = None, 0
            if lm.cross_attention:
                if req.cross is None:
                    raise ValueError("the model has cross attention: the request needs its condition [2, T, d]")
                cross = req.cross.to(lm.device, torch.float32).contiguous()
                if cross.dim() != 3 or cross.shape[0] != 2 or cross.shape[2] != lm.dim:
                    raise ValueError(f"cross must be [2, T, {lm.dim}] ([cond; null]), got {tuple(cross.shape)}")
                T = cross.shape[1]
                if not 1 <= T <= self.max_text:
                    raise ValueError(f"condition of {T} text positions: the session holds 1 .. {self.max_text}")
            prefix = req.prefix.to(lm.device, torch.float32).contiguous() if P else None
            F = req.prefill_cols
            if self.pages is None and F:
                _lib.check(lm._lib.acb_lm_admit_prompt(lm._handle, slot, _lib.ptr(cross), T, _lib.ptr(prefix), P, S, F,
                                                       C.c_uint64(req.seed), samp, None, 0, _lib.stream()), 'lm_admit_prompt')
            elif self.pages is None:
                _lib.check(lm._lib.acb_lm_admit_prefix(lm._handle, slot, _lib.ptr(cross), T, _lib.ptr(prefix), P, S,
                                                       C.c_uint64(req.seed), samp, _lib.stream()), 'lm_admit')
            else:
                ids = self.pages.take(slot, P + S)
                try:
                    pages = (C.c_int32 * len(ids))(*ids)
                    if F:
                        _lib.check(lm._lib.acb_lm_admit_prompt(lm._handle, slot, _lib.ptr(cross), T, _lib.ptr(prefix), P, S, F,
                                                               C.c_uint64(req.seed), samp, pages, len(ids), _lib.stream()),
                                   'lm_admit_prompt')
                    else:
                        _lib.check(lm._lib.acb_lm_admit_paged(lm._handle, slot, _lib.ptr(cross), T, _lib.ptr(prefix), P, S,
                                                              C.c_uint64(req.seed), samp, pages, len(ids), _lib.stream()),
                                   'lm_admit_paged')
                except Exception:
                    self.pages.release(slot)
                    raise
            # `keep`: the stream reads cross and the prefix after this call
            req.meta.update(S=S, mask=mask, pattern=pattern, keep=(cross, prefix))

    def retire(self, slot: int):
        """Cancel the slot's request between steps (acb_lm_retire): the slot stops decoding and is free for admission."""
        self._check_owner()
        with torch.cuda.device(self.lm.device):
            _lib.check(self.lm._lib.acb_lm_retire(self.lm._handle, slot, _lib.stream()), 'lm_retire')
        if self.pages is not None:
            self.pages.release(slot)

    def frames(self, slots: tp.List[int], t0: int, t1: int) -> torch.Tensor:
        """Codes [len(slots), K, t1 - t0] of frames [t0, t1) of the given slots, read from their delay-pattern sequences (frame t
        of codebook k is sequence step t + 1 + delays[k]); every frame must be final (below position - max_delay)."""
        lm = self.lm
        with torch.cuda.device(lm.device):
            t = torch.arange(t0, t1, device=lm.device)
            steps = t[None, :] + 1 + torch.tensor(self.delays, device=lm.device)[:, None]                # [K, n]
            idx = torch.tensor(slots, device=lm.device)
            return lm._bufs['seq'][idx].gather(2, steps[None].expand(len(slots), -1, -1))

    def steps(self, n: int):
        self._check_owner()
        with torch.cuda.device(self.lm.device):
            _lib.check(self.lm._lib.acb_lm_steps(self.lm._handle, n, _lib.stream()), 'lm_steps')

    def step_logits(self) -> torch.Tensor:
        """One step that also returns the CFG-mixed logits [slots, K, card] (rows of slots not decoding are not written)."""
        self._check_owner()
        lm = self.lm
        with torch.cuda.device(lm.device):
            out = torch.full((self.slots, lm.n_q, lm.card), float('nan'), device=lm.device, dtype=torch.float32)
            _lib.check(lm._lib.acb_lm_step_logits(lm._handle, out.data_ptr(), _lib.stream()), 'lm_step_logits')
            return out

    def status(self) -> tp.List[tp.Tuple[int, int]]:
        """[(position, status)] of every slot: one small device-to-host read."""
        self._check_owner()
        with torch.cuda.device(self.lm.device):
            _lib.check(self.lm._lib.acb_lm_slot_status(self.lm._handle, self._status.data_ptr(), _lib.stream()), 'lm_slot_status')
            return [tuple(r) for r in self._status.cpu().tolist()]

    def collect(self, slot: int, req: Request) -> torch.Tensor:
        """The finished request's codes [1, K, max_gen_len], prompt included.  Returns its pages to a paged session's pool."""
        lm, m = self.lm, req.meta
        with torch.cuda.device(lm.device):
            seq = lm._bufs['seq'][slot:slot + 1, :, :m['S']].clone()
            if self.pages is not None:
                self.pages.release(slot)
            return revert_sequence(lm, seq, m['mask'], m['pattern'], req.max_gen_len)


class ContinuousScheduler:
    """FIFO admission and retirement over a device session (`admit(slot, req)`, `steps(n)`, `status()`,
    `collect(slot, req)`, and `retire(slot)` for cancellation).  Every active slot advances one column per step, so the host
    knows when each one finishes: a poll admits waiting requests into free slots, runs steps up to the next retirement (at
    most `poll_steps`), checks the device status once, and returns the finished requests with their codes.  `last_admitted`
    holds the (slot, request) pairs the last poll admitted.

    On a paged session (one whose `pages` is a `PagePool`; `positions(req)` gives a request's length) the head of the queue is
    admitted only when a slot and its pages are free; while its pages are not, it waits and no later request overtakes it,
    so a long request is never starved by shorter ones.  `page_wait_steps` counts the steps run while the head waited for
    pages with a slot free, `page_steps` the pages in use summed over steps (mean: page_steps / steps_run).

    A request with prefilled prompt columns (`prefill_cols`) starts at that column.  A request longer than the session's
    window (`chain`, a `WindowChain`) is admitted as its first window; when a window finishes, the next one is admitted in the
    same poll into the same slot, ahead of every waiting request, and in a paged session it takes pages from those the
    finished window released (it never needs more).  The request is returned once, after its last window, with all its
    tokens.  `readmitted` counts those re-admissions."""

    def __init__(self, session, slots: int, poll_steps: tp.Optional[int] = None):
        if poll_steps is not None and poll_steps < 1:
            raise ValueError(f"poll_steps must be >= 1, got {poll_steps}")
        self.session, self.slots, self.poll_steps = session, slots, poll_steps
        self.waiting: tp.Deque[Request] = collections.deque()
        self.active: tp.Dict[int, Request] = {}
        self.pos: tp.Dict[int, int] = {}
        self.steps_run = 0
        self.busy_slot_steps = 0     # sum over steps of the active slots: occupancy = busy_slot_steps / (steps_run * slots)
        self.page_wait_steps = 0
        self.page_steps = 0
        self.last_admitted: tp.List[tp.Tuple[int, Request]] = []
        self.readmitted = 0

    def submit(self, req: Request):
        self.waiting.append(req)

    def cancel(self, request_id: int) -> bool:
        """Drop a waiting request, or retire an active one (its slot is free for the next poll).  False when the id is neither
        waiting nor decoding (finished, cancelled before or unknown)."""
        for req in self.waiting:
            if req.id == request_id:
                self.waiting.remove(req)
                return True
        for slot, req in self.active.items():
            if req.id == request_id:
                self.session.retire(slot)
                del self.active[slot]
                del self.pos[slot]
                return True
        return False

    @property
    def pending(self) -> bool:
        return bool(self.waiting or self.active)

    def _n_steps(self, req: Request) -> int:
        return req.meta['S'] - 1

    def poll(self) -> tp.List[tp.Tuple[Request, torch.Tensor]]:
        self.last_admitted = []
        pool = getattr(self.session, 'pages', None)
        waits = False
        for slot in range(self.slots):
            if not self.waiting:
                break
            if slot not in self.active:
                if pool is not None and not pool.fits(self.session.positions(self.waiting[0])):
                    waits = True
                    break
                req = self.waiting.popleft()
                self.session.admit(slot, req)
                self.active[slot] = req
                self.pos[slot] = req.prefill_cols
                self.last_admitted.append((slot, req))
        if not self.active:
            return []
        n = min(self._n_steps(r) - self.pos[s] for s, r in self.active.items())
        if self.poll_steps is not None:
            n = min(n, self.poll_steps)
        self.session.steps(n)
        self.steps_run += n
        self.busy_slot_steps += n * len(self.active)
        if pool is not None:
            self.page_steps += n * pool.in_use
            self.page_wait_steps += n if waits else 0
        status = self.session.status()
        done = []
        for slot in sorted(self.active):
            req = self.active[slot]
            self.pos[slot] += n
            pos, st = status[slot]
            finished = self.pos[slot] == self._n_steps(req)
            if pos != self.pos[slot] or st != (SLOT_FINISHED if finished else SLOT_ACTIVE):
                raise RuntimeError(f"slot {slot}: device at position {pos} status {st}, expected {self.pos[slot]} "
                                   f"{'finished' if finished else 'decoding'}")
            if finished:
                codes = self.session.collect(slot, req)
                nxt = req.chain.advance(codes) if req.chain is not None else None
                if nxt is not None:   # the request's next window, before any waiting request
                    assert self.session.positions(nxt) <= self.session.positions(req), \
                        "a later window needs more cache positions than the first"
                    assert pool is None or pool.fits(self.session.positions(nxt))
                    self.session.admit(slot, nxt)
                    self.active[slot] = nxt
                    self.pos[slot] = nxt.prefill_cols
                    self.readmitted += 1
                    continue
                done.append((req, codes if req.chain is None else req.chain.tokens()))
                del self.active[slot]
                del self.pos[slot]
        return done

    @property
    def occupancy(self) -> float:
        return self.busy_slot_steps / max(1, self.steps_run * self.slots)


class _Cohort:
    """Requests admitted in the same poll at the same start column: they advance in lock-step and share one stream decoder."""

    def __init__(self, members: tp.List[tp.Tuple[int, Request]], decoder, start: int, col0: int = 0):
        self.members, self.decoder = members, decoder
        self.start = start           # the scheduler's steps_run when the cohort was admitted
        self.col0 = col0             # the members' start column (their prefilled prompt columns)
        self.frames = 0              # frames handed to the decoder


class CohortStream:
    """Audio pieces of a session's requests while they decode, one codec call per cohort and poll.

    `stream_decoder(n)` makes a decoder over n items (`push(codes [n, K, m]) -> [n, C, m']`, `flush()`, `select(items)`).
    After a poll in which a request is at column c (its start column plus the steps it has run), its frames below
    c - max_delay are final (as in `LMModel.generate_blocks`), so a prefilled prompt's frames are final at admission and the
    requests admitted in one poll form one cohort per start column; the scheduler knows every position on the host, so nothing is read back to find them.  Each
    cohort's new frames go to its decoder in one push.  Members that finish are split out with `select` and flushed together
    (members of one cohort that finish in the same poll have the same length), the rest keep decoding in the remaining
    decoder.  A cancelled member is dropped from its cohort the same way.  `poll()` returns `(request_id, piece, tokens, final)`
    events: `piece` [1, C, m] is the request's next audio, `tokens` [1, K, n] the frames handed to the codec with it, and a
    request's pieces, concatenated, are the codec's decode of all its frames."""

    def __init__(self, scheduler: ContinuousScheduler, stream_decoder: tp.Callable[[int], tp.Any], max_delay: int):
        self.scheduler, self.stream_decoder, self.max_delay = scheduler, stream_decoder, max_delay
        self.cohorts: tp.List[_Cohort] = []
        self.codec_calls = 0         # pushes and flushes, over all polls

    def cancel(self, request_id: int) -> bool:
        if not self.scheduler.cancel(request_id):
            return False
        for co in self.cohorts:
            ids = [r.id for _, r in co.members]
            if request_id in ids:
                keep = [i for i, rid in enumerate(ids) if rid != request_id]
                if keep:
                    co.decoder = co.decoder.select(keep)
                    co.members = [co.members[i] for i in keep]
                else:
                    self.cohorts.remove(co)
                break
        return True

    def poll(self) -> tp.List[tp.Tuple[int, torch.Tensor, torch.Tensor, bool]]:
        sch = self.scheduler
        start = sch.steps_run
        done = sch.poll()
        by_col: tp.Dict[int, tp.List[tp.Tuple[int, Request]]] = {}
        for slot, req in sch.last_admitted:
            by_col.setdefault(req.prefill_cols, []).append((slot, req))
        for col0, members in by_col.items():
            self.cohorts.append(_Cohort(members, self.stream_decoder(len(members)), start, col0))
        finished = {req.id for req, _ in done}
        events = []
        for co in list(self.cohorts):
            events += self._advance(co, finished)
        return events

    def _advance(self, co: _Cohort, finished: tp.Set[int]) -> list:
        members = co.members
        fin = [i for i, (_, r) in enumerate(members) if r.id in finished]
        ready = max(0, co.col0 + self.scheduler.steps_run - co.start - self.max_delay)
        if ready == co.frames:   # no new frame, so no member finished either (its last step makes its last frame final)
            assert not fin
            return []
        codes = self.scheduler.session.frames([slot for slot, _ in members], co.frames, ready)
        wav = co.decoder.push(codes)
        co.frames = ready
        self.codec_calls += 1
        if fin:
            assert all(members[i][1].max_gen_len == ready for i in fin)
            keep = [i for i in range(len(members)) if i not in fin]
            if keep:
                tail = co.decoder.select(fin).flush()
                co.decoder = co.decoder.select(keep)
                co.members = [members[i] for i in keep]
            else:
                tail = co.decoder.flush()
                self.cohorts.remove(co)
            self.codec_calls += 1
        events = []
        for i, (_, req) in enumerate(members):
            piece = wav[i:i + 1]
            if i in fin:
                j = fin.index(i)
                piece = torch.cat([piece, tail[j:j + 1]], dim=-1)
            events.append((req.id, piece, codes[i:i + 1], i in fin))
        return events


class ContinuousGenerator:
    """`model.continuous(slots, poll_steps, max_text, return_tokens, chunk_duration)`: submit requests at any time, collect
    their audio as it decodes or when they finish.

    `submit(description=None, duration=None, prompt=None, prompt_sample_rate=None, *, melody=None, melody_sample_rate=None,
    use_sampling=None, top_k=None, top_p=None, temperature=None, cfg_coef=None)` returns a request id.  The sampling options are the request's own; None
    takes the value of `model.generation_params` when the generator was made.  Requests beyond `slots` wait in FIFO order.  A
    continuation prompt costs one decode step per prompt frame.  `cancel(request_id)` drops a waiting request or stops a
    decoding one, whose slot then takes the next waiting request; it returns False for a finished or unknown id, and a
    cancelled request yields nothing more.  `run()` polls until every submitted request has finished or been cancelled.

    Without `chunk_duration`, `poll()` runs one scheduling round and returns `(request_id, wav)` (or `(request_id, wav,
    tokens)` with return_tokens) for the requests that finished in it.  `wav` is [1, C, T] and `tokens` [1, K, T_frames]:
    what `generate([description])` (or `generate_continuation` / `generate_unconditional`) returns for that request alone,
    with its options, after the same `torch.manual_seed`.  On a melody model a request with `melody` ([C, T] or [1, C, T] at
    `melody_sample_rate`) returns what `generate_with_chroma([description], melody)` returns; without one its melody is
    null, as in `generate`.  Each request's chroma and description prefix is prefilled into its slot at admission.

    With `chunk_duration`, a round runs at most `round(chunk_duration * frame_rate)` steps and `poll()` returns
    `(request_id, piece, final)` (or `(request_id, piece, tokens, final)`) events: `piece` [1, C, m] is the request's next
    audio, as soon as the codec can produce it, and `final` marks its last event.  A request's pieces, concatenated, are the
    waveform the generator without chunk_duration returns for it; a continuation's first pieces are its prompt's audio.  The
    requests admitted in one round share one stream decoder.  Refused before any device work: a codec without a stream
    decoder (NotImplementedError) and chunk_duration <= 0 (ValueError).

    With `kv_cache_gb`, the session is paged (`SlotSession(kv_pages=...)`): its self-attention KV cache is a pool of
    floor(kv_cache_gb * 1e9 / kv_page_bytes) pages, each request holds only the pages its own length needs, and a request
    waits in FIFO order until a slot and its pages are free.  Refused before any device work: kv_cache_gb <= 0, and a budget
    that cannot hold one request of max_duration (ValueError).  Results are those of the session without kv_cache_gb.

    With `kv_cache_dtype='fp8'` (default 'fp16'; needs kv_cache_gb) the pool holds e4m3 codes and one fp32 scale per
    position and head (`SlotSession(kv_dtype='fp8')`), so the same budget holds about 1.88x the pages.  Results then equal
    the same request alone in an fp8 session, not `generate` or the fp16 session.  Refused before any device work: another
    kv_cache_dtype, and 'fp8' without kv_cache_gb (ValueError).

    With `prefill_prompts`, a request's results are those of `generate`'s default path instead of ``ACB_LM_PREFILL=0``: its
    prompt columns [0, first) (first as `LMModel.generate` computes it, `prefill_columns`) are prefilled into its slot at
    admission (acb_lm_admit_prompt), in the passes `generate` runs for it alone, and the slot decodes from column `first`.
    A continuation then occupies its slot `first` fewer steps, but its passes (32 positions each) run between two steps, so
    every other slot waits for them: prefill lowers a prompted request's latency and can cost the session's throughput when
    many slots are busy.  It also serves durations beyond max_duration, window by window as `generate` does
    (`musicgen.window_plan`, `extend_stride` of the model's generation parameters): each window after the first is admitted
    into the same slot as soon as the previous one finishes, with the previous window's tail prefilled as its prompt, and on a
    melody model with the melody re-sliced from the window's offset.  `submit` draws one seed per window, in `generate`'s
    order.  A long request is returned once, with all its frames; it is refused with `chunk_duration` (NotImplementedError),
    as a stream decoder is not carried from one window to the next.

    Refused before any device work: durations beyond max_duration without prefill_prompts, two_step_cfg and cfg_coef_beta
    (NotImplementedError), a melody on a model without a melody conditioner (NotImplementedError), a melody together with a
    prompt, and a description longer than max_text text positions (ValueError)."""

    prefill_prompts = False
    DECODE_GROUP = 32   # requests per codec call in poll()

    def __init__(self, model, slots: int = 32, poll_steps: tp.Optional[int] = None, max_text: int = 64,
                 return_tokens: bool = False, chunk_duration: tp.Optional[float] = None,
                 kv_cache_gb: tp.Optional[float] = None, prefill_prompts: bool = False, kv_cache_dtype: str = 'fp16'):
        params = dict(model.generation_params)
        check_kv_dtype(kv_cache_dtype)
        if kv_cache_dtype == 'fp8' and kv_cache_gb is None:
            raise ValueError("kv_cache_dtype='fp8' is built for the paged KV cache only: pass kv_cache_gb")
        kv_pages = None if kv_cache_gb is None else kv_pages_for_budget(model.lm, kv_cache_gb, kv_cache_dtype)
        if getattr(model, '_has_melody', False) != model.lm.has_prefix:
            raise NotImplementedError("continuous batching takes a melody ('self_wav') conditioner only as a condition prefix "
                                      "(prepend fuser), and a condition prefix only from one")
        if params.get('two_step_cfg'):
            raise NotImplementedError("continuous batching with two_step_cfg is not built")
        if params.get('cfg_coef_beta') is not None:
            raise NotImplementedError("continuous batching with cfg_coef_beta (double CFG) is not built")
        if chunk_duration is not None:
            if not chunk_duration > 0:
                raise ValueError(f"chunk_duration must be > 0, got {chunk_duration}")
            if not hasattr(model.compression_model, 'stream_decoder'):
                raise NotImplementedError(f"{type(model.compression_model).__name__} has no stream decoder")
            model.compression_model.stream_decoder(1)   # GroupNorm and transformers' chunked codecs refuse here
            block = max(1, int(round(chunk_duration * model.frame_rate)))
            poll_steps = block if poll_steps is None else min(poll_steps, block)
        self.model, self.return_tokens, self.prefill_prompts = model, return_tokens, bool(prefill_prompts)
        self.defaults = dict(use_sampling=params['use_sampling'], temp=params['temp'], top_k=params['top_k'],
                             top_p=params['top_p'], cfg_coef=params['cfg_coef'])
        max_gen_len = int(model.max_duration * model.frame_rate)
        self.session = SlotSession(model.lm, slots, max_gen_len, max_text, **self.defaults, kv_pages=kv_pages,
                                   kv_dtype=kv_cache_dtype)
        self.scheduler = ContinuousScheduler(self.session, slots, poll_steps)
        self.stream = None
        if chunk_duration is not None:
            self.stream = CohortStream(self.scheduler, model.compression_model.stream_decoder, self.session.max_delay)
        self._ids = itertools.count()
        self._cancelled: tp.Set[int] = set()

    def submit(self, description: tp.Optional[str] = None, duration: tp.Optional[float] = None,
               prompt: tp.Optional[torch.Tensor] = None, prompt_sample_rate: tp.Optional[int] = None, *,
               melody: tp.Optional[torch.Tensor] = None, melody_sample_rate: tp.Optional[int] = None,
               use_sampling: tp.Optional[bool] = None, top_k: tp.Optional[int] = None, top_p: tp.Optional[float] = None,
               temperature: tp.Optional[float] = None, cfg_coef: tp.Optional[float] = None) -> int:
        from .audio_utils import convert_audio
        m = self.model
        duration = m.duration if duration is None else float(duration)
        long = duration > m.max_duration
        if long and not self.prefill_prompts:
            raise NotImplementedError(f"duration {duration} > max_duration {m.max_duration}: window extension needs a session "
                                      "with prefill_prompts=True")
        if long and self.stream is not None:
            raise NotImplementedError(f"duration {duration} > max_duration {m.max_duration} with chunk_duration: streaming a "
                                      "request across windows is not built")
        n = int(duration * m.frame_rate)
        if n < 1:
            raise ValueError(f"duration {duration} s is less than one frame")
        if prompt is not None:
            if prompt_sample_rate is None:
                raise ValueError("prompt_sample_rate is required with a prompt")
            if prompt.dim() == 2:
                prompt = prompt[None]
            if prompt.dim() != 3 or prompt.shape[0] != 1:
                raise ValueError("prompt should be one item: [C, T] or [1, C, T]")
        if melody is not None:
            if not getattr(m, '_has_melody', False):
                raise NotImplementedError("this model has no melody ('self_wav') conditioner; use a MusicGen-melody model")
            if prompt is not None:
                raise ValueError("a melody and a prompt together: generate_with_chroma takes no prompt")
            if melody_sample_rate is None:
                raise ValueError("melody_sample_rate is required with a melody")
            if melody.dim() == 3 and melody.shape[0] == 1:
                melody = melody[0]
            if melody.dim() != 2:
                raise ValueError("melody should be one item: [C, T] or [1, C, T]")
        given = dict(use_sampling=use_sampling, temp=temperature, top_k=top_k, top_p=top_p, cfg_coef=cfg_coef)
        options = {k: self.defaults[k] if v is None else v for k, v in given.items()}
        if options['cfg_coef'] is None:
            options['cfg_coef'] = m.lm.cfg_coef
        check_sampling(**options)
        if prompt is not None:
            prompt = convert_audio(prompt, prompt_sample_rate, m.sample_rate, m.audio_channels)
        if melody is not None:
            attributes, prompt_tokens = m._prepare_melody([description], [melody], melody_sample_rate)
        else:   # on a melody model every item carries a melody condition: a null one here
            attributes, prompt_tokens = m._prepare_tokens_and_attributes([description], prompt)
        T0 = 0 if prompt_tokens is None else prompt_tokens.shape[-1]
        plan = window_plan(duration, m.max_duration, m.extend_stride, m.frame_rate, T0) if long else None
        first_len = plan[0].length if long else n
        if prompt_tokens is not None and T0 >= first_len:
            raise ValueError(f"the prompt ({T0} frames) must be shorter than the generation ({first_len})")
        # a long request's windows in generate's order: window k's conditions (a melody re-sliced from its offset), then
        # its seed, drawn as LMModel.generate draws it
        windows = []
        for k in range(len(plan) if long else 1):
            if k == 0 or getattr(m, '_has_melody', False):   # a text condition is the same in every window
                attrs = m._window_attributes(attributes, plan[k].time_offset) if long else attributes
                cross, prefix = self._conditions(attrs)
            windows.append((cross, prefix, int(torch.randint(0, 2 ** 62, (1,)).item())))
        rid = next(self._ids)

        def make(k: int, prompt: tp.Optional[torch.Tensor]) -> Request:
            length = plan[k].length if long else n
            cols = prefill_columns(m.lm, prompt.shape[-1], length) if self.prefill_prompts and prompt is not None else 0
            cross, prefix, seed = windows[k]
            return Request(length, cross, prompt, seed, rid, **options, prefix=prefix, prefill_cols=cols, chain=chain)

        chain = WindowChain(plan, make, prompt_tokens) if long else None
        self.scheduler.submit(make(0, prompt_tokens))
        return rid

    def _conditions(self, attributes):
        """A request's cross [2, T, d] and prefix [2, P, d] (None where the model has none), checked against the session."""
        m = self.model
        cross = prefix = None
        if m.lm.cross_attention or m.lm.has_prefix:
            cross, prefix = m.lm._condition_tensors(attributes)
            cross = cross if m.lm.cross_attention else None
        if cross is not None and cross.shape[1] > self.session.max_text:
            raise ValueError(f"the description has {cross.shape[1]} text positions; the session holds {self.session.max_text}")
        if prefix is not None and prefix.shape[1] > self.session.max_prefix:
            raise ValueError(f"the condition prefix has {prefix.shape[1]} positions (chroma and description); the session holds "
                             f"{self.session.max_prefix}: the description is longer than {self.session.max_text} text positions")
        return cross, prefix

    def cancel(self, request_id: int) -> bool:
        """Drop a waiting request or stop a decoding one (acb_lm_retire); False for a finished or unknown id."""
        ok = self.stream.cancel(request_id) if self.stream is not None else self.scheduler.cancel(request_id)
        if ok:
            self._cancelled.add(request_id)
        return ok

    @property
    def pending(self) -> bool:
        return self.scheduler.pending

    @property
    def occupancy(self) -> float:
        return self.scheduler.occupancy

    def poll(self) -> tp.List[tuple]:
        if self.stream is not None:
            out = []
            for rid, piece, tokens, final in self.stream.poll():
                if piece.shape[-1] or final or self.return_tokens:
                    out.append((rid, piece, tokens, final) if self.return_tokens else (rid, piece, final))
            return out
        done = self.scheduler.poll()
        out = {}
        by_len: tp.Dict[int, tp.List[tp.Tuple[Request, torch.Tensor]]] = collections.defaultdict(list)
        for req, tokens in done:
            by_len[tokens.shape[-1]].append((req, tokens))
        for same_len in by_len.values():   # the items that finished together and have one length: one codec call per
            # DECODE_GROUP of them, so a wide session whose requests finish together (128 slots of 30 s) does not hold the
            # codec's activations for all of them at once
            for g0 in range(0, len(same_len), self.DECODE_GROUP):
                group = same_len[g0:g0 + self.DECODE_GROUP]
                tokens = torch.cat([t for _, t in group], dim=0)
                wav = self.model.generate_audio(tokens)
                for i, (req, tok) in enumerate(group):
                    out[req.id] = (req.id, wav[i:i + 1], tok) if self.return_tokens else (req.id, wav[i:i + 1])
        return [out[req.id] for req, _ in done]

    def run(self) -> tp.Iterator[tuple]:
        while self.pending:
            for ev in self.poll():
                if ev[0] not in self._cancelled:   # a request cancelled while this round's events are consumed
                    yield ev
