"""Streaming SEANet decode: the per-layer context and lookahead arithmetic, free of kernel calls.

`DecoderStream` runs the decoder's layer plan (`synth.encodec_layers(cfg)['decoder']`) over a latent that arrives in pieces and
returns, after each piece, every output sample that no later frame can change.  It only slices and joins tensors; the layers
themselves run through a backend with four operations, each on a window that needs no padding:

    conv(L, x)                        valid convolution of layer L (ELU on its input when L says so), stride L['stride']
    resblock(block, x, pad_left)      one SEANetResnetBlock (shortcut, conv k, conv 1x1) on the valid window x; the skip is x's
                                      steps [pad_left, pad_left + n_out)
    convtr(L, x, trim_left, t_out)    transposed conv of L with x[-1] = x[t_in] = 0, full-output steps [trim_left, trim_left + t_out)
    lstm(L, x, state)                 the LSTM block (y = LSTM(x) + x) from `state`, which it advances; lstm_state(L, batch) makes one
                                      and lstm_select(L, state, items) copies the given items of one (only `select` needs it)

`EncodecModel.stream_decoder` plugs in the CUDA kernels; the CPU tests plug in the oracle's layers.

What each layer keeps (reference semantics: audiocraft/modules/conv.py:185-243, seanet.py):
  * a convolution of effective kernel k_eff and stride s keeps the padded input its next output needs, k_eff - s steps in
    steady state.  The first window gets the left padding; the right padding, with get_extra_padding_for_conv1d's extra steps,
    is appended at flush from the total length, exactly as `decode` pads the whole sequence.  A reflect pad reaches
    max(pad_left, pad_right) + 1 steps into the sequence (pad1d pads shorter inputs with zeros first), so a reflect-padded layer
    waits for that many steps before its first output, and at flush a layer that never started pads its whole input at once;
  * a transposed conv (kernel 2 * stride) keeps the previous input step: full-output step u depends on inputs u // s and
    u // s - 1, so after n inputs the steps below n * s are final and the last s come at flush (x[n] = 0);
  * the LSTM keeps (h, c) per layer.
"""
import copy
import math
import typing as tp

import torch


def _extra_padding(length: int, k_eff: int, stride: int, padding_total: int) -> int:
    """get_extra_padding_for_conv1d, audiocraft/modules/conv.py:47-53."""
    n_frames = (length - k_eff + padding_total) / stride + 1
    return (math.ceil(n_frames) - 1) * stride + (k_eff - padding_total) - length


def _pad1d(x: torch.Tensor, left: int, right: int, reflect: bool) -> torch.Tensor:
    """pad1d, audiocraft/modules/conv.py:71-88: a reflect pad first zero-extends an input no longer than the pad."""
    if not reflect:
        return torch.nn.functional.pad(x, (left, right))
    length, big, grow = x.shape[-1], max(left, right), 0
    if length <= big:
        grow = big - length + 1
        x = torch.nn.functional.pad(x, (0, grow))
    y = torch.nn.functional.pad(x, (left, right), 'reflect')
    return y[..., :y.shape[-1] - grow]


def _cat(a: tp.Optional[torch.Tensor], b: tp.Optional[torch.Tensor]) -> tp.Optional[torch.Tensor]:
    if a is None or a.shape[-1] == 0:
        return b
    if b is None or b.shape[-1] == 0:
        return a
    return torch.cat([a, b], dim=-1)


class _ConvStage:
    """A convolution, or a residual block whose geometry is its k-tap convolution's (the 1x1 convolutions need no context)."""

    def __init__(self, run, k_eff: int, stride: int, causal: bool, reflect: bool):
        self.run, self.k_eff, self.s, self.reflect = run, k_eff, stride, reflect
        total = k_eff - stride
        self.pr0 = 0 if causal else total // 2
        self.pl = total - self.pr0
        self.pr_max = self.pr0 + stride - 1            # the extra padding is at most stride - 1 steps
        self.total = total
        self.n_in = 0                                  # raw input steps received
        self.pending: tp.Optional[torch.Tensor] = None # raw input held before the first window (reflect pads)
        self.buf: tp.Optional[torch.Tensor] = None     # padded input from padded step p0 on
        self.p0 = 0
        self.j = 0                                     # next output step

    def last_in(self, o: int) -> int:
        return o * self.s - self.pl + self.k_eff - 1

    def _emit(self) -> tp.Optional[torch.Tensor]:
        end = self.p0 + self.buf.shape[-1]
        j_end = (end - self.k_eff) // self.s + 1 if end >= self.k_eff else 0
        y = None
        if j_end > self.j:
            a = self.j * self.s - self.p0
            y = self.run(self.buf[..., a:a + (j_end - 1 - self.j) * self.s + self.k_eff], self.pl)
            self.j = j_end
        keep = self.j * self.s
        if self.reflect:                               # the right reflect pad reads the last pr + 1 raw steps
            keep = min(keep, self.pl + self.n_in - (self.pr_max + 1))
        keep = max(keep, self.p0)
        self.buf = self.buf[..., keep - self.p0:]
        self.p0 = keep
        return y

    def push(self, x: tp.Optional[torch.Tensor]) -> tp.Optional[torch.Tensor]:
        if x is None or x.shape[-1] == 0:
            return None
        self.n_in += x.shape[-1]
        if self.buf is None:
            self.pending = _cat(self.pending, x)
            if self.reflect and self.n_in <= max(self.pl, self.pr_max):
                return None
            p = self.pending
            left = p[..., 1:self.pl + 1].flip(-1) if self.reflect else p.new_zeros(p.shape[:-1] + (self.pl,))
            self.buf, self.pending = torch.cat([left, p], dim=-1), None
        else:
            self.buf = torch.cat([self.buf, x], dim=-1)
        return self._emit()

    def select(self, items: tp.List[int]) -> '_ConvStage':
        out = copy.copy(self)
        out.pending = None if self.pending is None else self.pending[items]
        out.buf = None if self.buf is None else self.buf[items]
        return out

    def flush(self) -> tp.Optional[torch.Tensor]:
        if self.n_in == 0:
            return None
        pr = self.pr0 + _extra_padding(self.n_in, self.k_eff, self.s, self.total)
        if self.buf is None:
            self.buf, self.pending = _pad1d(self.pending, self.pl, pr, self.reflect), None
        elif self.reflect:
            a = self.pl + self.n_in - 1 - pr - self.p0
            self.buf = torch.cat([self.buf, self.buf[..., a:a + pr].flip(-1)], dim=-1)
        else:
            self.buf = torch.nn.functional.pad(self.buf, (0, pr))
        y = self._emit()
        assert self.j == (self.n_in + self.pl + pr - self.k_eff) // self.s + 1
        return y


class _ConvTrStage:
    def __init__(self, run, kernel: int, stride: int, causal: bool, trim_right_ratio: float):
        assert kernel == 2 * stride, 'the streaming transposed conv is built for kernel == 2 * stride (every SEANet decoder)'
        total = kernel - stride
        self.right = math.ceil(total * trim_right_ratio) if causal else total // 2
        self.left = total - self.right
        self.run, self.s = run, stride
        self.prev: tp.Optional[torch.Tensor] = None

    def last_in(self, o: int) -> int:
        return (o + self.left) // self.s

    def push(self, x: tp.Optional[torch.Tensor]) -> tp.Optional[torch.Tensor]:
        if x is None or x.shape[-1] == 0:
            return None
        n = x.shape[-1]
        if self.prev is None:
            y = self.run(x, self.left, n * self.s - self.left) if n * self.s > self.left else None
        else:
            y = self.run(torch.cat([self.prev, x], dim=-1), self.s, n * self.s)
        self.prev = x[..., -1:]
        return y

    def select(self, items: tp.List[int]) -> '_ConvTrStage':
        out = copy.copy(self)
        out.prev = None if self.prev is None else self.prev[items]
        return out

    def flush(self) -> tp.Optional[torch.Tensor]:
        if self.prev is None or self.s == self.right:
            return None
        return self.run(self.prev, self.s, self.s - self.right)


class _LstmStage:
    def __init__(self, run, state, pick):
        self.run, self.state, self.pick = run, state, pick

    def select(self, items: tp.List[int]) -> '_LstmStage':
        return _LstmStage(self.run, self.pick(self.state, items), self.pick)

    def last_in(self, o: int) -> int:
        return o

    def push(self, x):
        if x is None or x.shape[-1] == 0:
            return None
        return self.run(x, self.state)

    def flush(self):
        return None


def decoder_blocks(layers: tp.List[dict]) -> tp.List[tp.Tuple[str, tp.Any]]:
    """The decoder plan grouped into ('conv', L), ('convtr', L), ('lstm', L) and ('block', (shortcut or None, conv k, conv 1x1))."""
    out, i = [], 0
    while i < len(layers):
        L = layers[i]
        if L['kind'] == 'conv' and L['res'] == 'shortcut':
            out.append(('block', (L, layers[i + 1], layers[i + 2])))
            i += 3
        elif L['kind'] == 'conv' and L['res'] == 'in':
            out.append(('block', (None, L, layers[i + 1])))
            i += 2
        else:
            out.append((L['kind'], L))
            i += 1
    for kind, b in out:
        if kind == 'block':
            assert b[1]['stride'] == 1 and b[2]['k'] == 1 and b[2]['res'] == 'out' and (b[0] is None or b[0]['k'] == 1), b
    return out


class DecoderStream:
    """The SEANet decoder over a latent [B, D, n] pushed in pieces.  `push(z)` returns the newly final samples (None when there
    are none yet), `flush()` the rest; their concatenation is the decoder's output on the whole latent, extra padding included."""

    def __init__(self, layers: tp.List[dict], cfg: dict, backend, batch: int):
        causal, reflect = bool(cfg['causal']), cfg['pad_mode'] == 'reflect'
        self.hop = math.prod(cfg['ratios'])
        self.stages: tp.List[tp.Any] = []
        for kind, L in decoder_blocks(layers):
            if kind == 'conv':
                k_eff = (L['k'] - 1) * L['dilation'] + 1
                self.stages.append(_ConvStage(lambda x, pl, L=L: backend.conv(L, x), k_eff, L['stride'], causal, reflect))
            elif kind == 'block':
                a = L[1]
                k_eff = (a['k'] - 1) * a['dilation'] + 1
                self.stages.append(_ConvStage(lambda x, pl, L=L: backend.resblock(L, x, pl), k_eff, 1, causal, reflect))
            elif kind == 'convtr':
                self.stages.append(_ConvTrStage(lambda x, tl, n, L=L: backend.convtr(L, x, tl, n), L['k'], L['stride'], causal,
                                                cfg['trim_right_ratio']))
            else:
                self.stages.append(_LstmStage(lambda x, st, L=L: backend.lstm(L, x, st), backend.lstm_state(L, batch),
                                              lambda st, items, L=L: backend.lstm_select(L, st, items)))

    @property
    def lookahead(self) -> int:
        """Frames past its own a sample waits for once the stream is running: the largest F(o) - o // hop, with F(o) the last latent
        frame output sample o depends on.  (A reflect pad's first window reaches further, see the module docstring.)"""
        o0 = 64 * self.hop
        best = 0
        for o in range(o0, o0 + self.hop):
            f = o
            for st in reversed(self.stages):
                f = st.last_in(f)
            best = max(best, f - o // self.hop)
        return best

    def select(self, items: tp.List[int]) -> 'DecoderStream':
        """A stream of the given items only (indices into the batch, in that order), in the same state: every stage's held
        input, the transposed convolutions' previous step and the LSTM state are copied along the batch.  The items' output
        continues exactly as in this stream; this stream is unchanged."""
        out = copy.copy(self)
        out.stages = [st.select(items) for st in self.stages]
        return out

    def push(self, z: torch.Tensor) -> tp.Optional[torch.Tensor]:
        x = z
        for st in self.stages:
            x = st.push(x)
        return x

    def flush(self) -> tp.Optional[torch.Tensor]:
        x = None
        for st in self.stages:
            x = _cat(st.push(x), st.flush())
        return x
