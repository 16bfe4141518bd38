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
forcing), which costs one step per prompt column, where `generate` prefills it several positions per pass.

`ContinuousScheduler` is the host-side policy (FIFO admission, retirement) over any object with the device session's four
methods, so it is tested without a GPU; `ContinuousGenerator` (``BaseGenModel.continuous``) is the public entry point.
"""
import collections
import ctypes as C
import itertools
import typing as tp
from dataclasses import dataclass, field

import torch

from . import _lib

SLOT_INACTIVE, SLOT_ACTIVE, SLOT_FINISHED = 0, 1, 2


@dataclass
class Request:
    """One generation request at the LM level: cross [2, T, d] ([cond; null]) or None, prompt codes [1, K, T0] or None."""
    max_gen_len: int
    cross: tp.Optional[torch.Tensor] = None
    prompt: tp.Optional[torch.Tensor] = None
    seed: int = 0
    id: int = -1
    meta: tp.Dict[str, tp.Any] = field(default_factory=dict)   # filled by the session at admission


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
    (slot s owns rows s and slots + s).  Holds the model's decode handle until another generation call takes it."""

    def __init__(self, lm, slots: int, max_gen_len: int, max_text: int = 64, use_sampling: bool = True, temp: float = 1.0,
                 top_k: int = 250, top_p: float = 0.0, cfg_coef: tp.Optional[float] = None):
        if not 1 <= slots <= _lib.ACB_LM_MAX_SLOTS:
            raise ValueError(f"slots must be in [1, {_lib.ACB_LM_MAX_SLOTS}], got {slots}")
        if max_gen_len < 1 or max_text < 1:
            raise ValueError("max_gen_len and max_text must be >= 1")
        if lm.has_prefix:
            raise NotImplementedError("continuous batching with a condition prefix (prepend fuser, melody) is not built")
        self.lm, self.slots, self.max_gen_len, self.max_text = lm, slots, max_gen_len, max_text
        self.seq_len_max = pattern_sequence(lm, None, max_gen_len)[0].shape[-1]
        coef = lm.cfg_coef if cfg_coef is None else cfg_coef
        with torch.cuda.device(lm.device):
            lm._ensure(2 * slots, self.seq_len_max, max_text if lm.cross_attention else 0, slots)
            samp = _lib.LMSampling(int(bool(use_sampling)), float(temp), int(top_k), float(top_p), float(coef), 0, 0, 0.0)
            _lib.check(lm._lib.acb_lm_begin_slots(lm._handle, slots, max_text, self.seq_len_max, C.byref(samp),
                                                  _lib.stream()), 'lm_begin_slots')
            lm.launches_per_step = lm._lib.acb_lm_launches_per_step(lm._handle)
            lm._session = self
            self._status = torch.zeros((slots, 2), device=lm.device, dtype=torch.int32)

    def _check_owner(self):
        if self.lm._session is not self:
            raise RuntimeError("the LM's decode handle was taken by another generation call; start a new session")

    def admit(self, slot: int, req: Request):
        """Write the request's sequence and mask rows, then its cross K/V and slot state (acb_lm_admit)."""
        self._check_owner()
        lm = self.lm
        if req.max_gen_len > self.max_gen_len:
            raise ValueError(f"max_gen_len {req.max_gen_len} > the session's {self.max_gen_len}")
        with torch.cuda.device(lm.device):
            seq, mask, pattern = pattern_sequence(lm, req.prompt, req.max_gen_len, lm.device)
            S = seq.shape[-1]
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
            _lib.check(lm._lib.acb_lm_admit(lm._handle, slot, _lib.ptr(cross), T, S, C.c_uint64(req.seed), _lib.stream()),
                       'lm_admit')
            req.meta.update(S=S, mask=mask, pattern=pattern, keep=cross)   # `keep`: the stream reads cross after this call

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
        """The finished request's codes [1, K, max_gen_len], prompt included."""
        lm, m = self.lm, req.meta
        with torch.cuda.device(lm.device):
            seq = lm._bufs['seq'][slot:slot + 1, :, :m['S']].clone()
            return revert_sequence(lm, seq, m['mask'], m['pattern'], req.max_gen_len)


class ContinuousScheduler:
    """FIFO admission and retirement over a device session (`admit(slot, req)`, `steps(n)`, `status()`,
    `collect(slot, req)`).  Every active slot advances one column per step, so the host knows when each one finishes: a poll
    admits waiting requests into free slots, runs steps up to the next retirement (at most `poll_steps`), checks the device
    status once, and returns the finished requests with their codes."""

    def __init__(self, session, slots: int, poll_steps: tp.Optional[int] = None):
        if poll_steps is not None and poll_steps < 1:
            raise ValueError(f"poll_steps must be >= 1, got {poll_steps}")
        self.session, self.slots, self.poll_steps = session, slots, poll_steps
        self.waiting: tp.Deque[Request] = collections.deque()
        self.active: tp.Dict[int, Request] = {}
        self.pos: tp.Dict[int, int] = {}
        self.steps_run = 0
        self.busy_slot_steps = 0     # sum over steps of the active slots: occupancy = busy_slot_steps / (steps_run * slots)

    def submit(self, req: Request):
        self.waiting.append(req)

    @property
    def pending(self) -> bool:
        return bool(self.waiting or self.active)

    def _n_steps(self, req: Request) -> int:
        return req.meta['S'] - 1

    def poll(self) -> tp.List[tp.Tuple[Request, torch.Tensor]]:
        for slot in range(self.slots):
            if not self.waiting:
                break
            if slot not in self.active:
                req = self.waiting.popleft()
                self.session.admit(slot, req)
                self.active[slot] = req
                self.pos[slot] = 0
        if not self.active:
            return []
        n = min(self._n_steps(r) - self.pos[s] for s, r in self.active.items())
        if self.poll_steps is not None:
            n = min(n, self.poll_steps)
        self.session.steps(n)
        self.steps_run += n
        self.busy_slot_steps += n * len(self.active)
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
                done.append((req, self.session.collect(slot, req)))
                del self.active[slot]
                del self.pos[slot]
        return done

    @property
    def occupancy(self) -> float:
        return self.busy_slot_steps / max(1, self.steps_run * self.slots)


class ContinuousGenerator:
    """`model.continuous(slots, poll_steps)`: submit requests at any time, collect waveforms as they finish.

    `submit(description=None, duration=None, prompt=None, prompt_sample_rate=None)` returns a request id; `poll()` runs one
    scheduling round and returns the `(request_id, wav)` (or `(request_id, wav, tokens)` with return_tokens) of the requests
    that finished in it, `run()` polls until every submitted request has finished.  `wav` is [1, C, T] and `tokens`
    [1, K, T_frames]: what `generate([description])` (or `generate_continuation` / `generate_unconditional`) returns for that
    request alone after the same `torch.manual_seed`.  Requests beyond `slots` wait in FIFO order.  A continuation prompt costs
    one decode step per prompt frame.  Refused (NotImplementedError, before any device work): durations beyond
    max_duration, melody models, two_step_cfg and cfg_coef_beta."""

    def __init__(self, model, slots: int = 32, poll_steps: tp.Optional[int] = None, max_text: int = 64,
                 return_tokens: bool = False):
        params = dict(model.generation_params)
        if getattr(model, '_has_melody', False) or model.lm.has_prefix:
            raise NotImplementedError("continuous batching of melody-conditioned models (a condition prefix) is not built")
        if params.get('two_step_cfg'):
            raise NotImplementedError("continuous batching with two_step_cfg is not built")
        if params.get('cfg_coef_beta') is not None:
            raise NotImplementedError("continuous batching with cfg_coef_beta (double CFG) is not built")
        self.model, self.return_tokens = model, return_tokens
        max_gen_len = int(model.max_duration * model.frame_rate)
        self.session = SlotSession(model.lm, slots, max_gen_len, max_text, use_sampling=params['use_sampling'],
                                   temp=params['temp'], top_k=params['top_k'], top_p=params['top_p'],
                                   cfg_coef=params['cfg_coef'])
        self.scheduler = ContinuousScheduler(self.session, slots, poll_steps)
        self._ids = itertools.count()

    def submit(self, description: tp.Optional[str] = None, duration: tp.Optional[float] = None,
               prompt: tp.Optional[torch.Tensor] = None, prompt_sample_rate: tp.Optional[int] = None) -> int:
        from .audio_utils import convert_audio
        m = self.model
        duration = m.duration if duration is None else float(duration)
        if duration > m.max_duration:
            raise NotImplementedError(f"duration {duration} > max_duration {m.max_duration}: window extension is not built "
                                      "for continuous batching")
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
            prompt = convert_audio(prompt, prompt_sample_rate, m.sample_rate, m.audio_channels)
        attributes, prompt_tokens = m._prepare_tokens_and_attributes([description], prompt)
        if prompt_tokens is not None and prompt_tokens.shape[-1] >= n:
            raise ValueError(f"the prompt ({prompt_tokens.shape[-1]} frames) must be shorter than the generation ({n})")
        cross = m.lm._condition_tensors(attributes)[0] if m.lm.cross_attention else None
        if cross is not None and cross.shape[1] > self.session.max_text:
            raise ValueError(f"the description has {cross.shape[1]} text positions; the session holds {self.session.max_text}")
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())   # drawn as LMModel.generate draws it
        rid = next(self._ids)
        self.scheduler.submit(Request(n, cross, prompt_tokens, seed, rid))
        return rid

    @property
    def pending(self) -> bool:
        return self.scheduler.pending

    @property
    def occupancy(self) -> float:
        return self.scheduler.occupancy

    def poll(self) -> tp.List[tuple]:
        done = self.scheduler.poll()
        out = {}
        by_len: tp.Dict[int, tp.List[tp.Tuple[Request, torch.Tensor]]] = collections.defaultdict(list)
        for req, tokens in done:
            by_len[tokens.shape[-1]].append((req, tokens))
        for group in by_len.values():   # the items that finished together and have one length: one codec call
            tokens = torch.cat([t for _, t in group], dim=0)
            wav = self.model.generate_audio(tokens)
            for i, (req, tok) in enumerate(group):
                out[req.id] = (req.id, wav[i:i + 1], tok) if self.return_tokens else (req.id, wav[i:i + 1])
        return [out[req.id] for req, _ in done]

    def run(self) -> tp.Iterator[tuple]:
        while self.pending:
            yield from self.poll()
