"""Layer-window pipeline over torch.distributed — prima.cpp's piped ring (src/llama.cpp:3838-3883 this_layer_is_mine /
map_layer_to_local_id, llama_send/recv_tensors :18031-18077) re-targeted to the GPUs of one NVSwitch box.

One process per GPU.  Rank r owns the contiguous layers [bounds[r], bounds[r+1]); rank 0 also owns the token embedding, the
last rank owns output_norm + lm_head.  Per token there is exactly ONE point-to-point hand-off of the hidden state
[n_embd] f32 per stage boundary (NCCL send/recv over NVLink; the reference ships the same f32 payload over ZeroMQ/TCP), and
the sampled token id returns from the last rank to rank 0 (prima returns the result to the master, :18559-18563), which keeps
decoding strictly sequential.  No collective is involved: the path has no reduction step.

The stage object only needs: decode_async(token, pos), and the tensors hidden_in / hidden_out / logits that alias the
engine's device buffers.  The same class drives CPU tensors over gloo in the tests.

Stream contract: NCCL orders its transfers against torch's CURRENT stream, the engine enqueues on its own stream (pb200_stream).  Pass
that stream (a torch.cuda.ExternalStream over it) as `stream=` and the runners enter it around every exchange + step themselves; without
it the caller must have made it current (bench.py does both)."""
from __future__ import annotations

import contextlib


def _entered(stream):
    """Context manager that makes `stream` torch's current stream (no-op for None / CPU runs)."""
    if stream is None:
        return contextlib.nullcontext()
    import torch
    return torch.cuda.stream(stream)


def layer_windows(n_layer: int, world: int) -> list[int]:
    """Uniform contiguous windows (8 identical GPUs need no ILP scheduler, common/common.cpp:860-1594): bounds[r]..bounds[r+1]."""
    if world < 1 or n_layer < world:
        raise ValueError("need 1 <= world <= n_layer")
    return [round(r * n_layer / world) for r in range(world + 1)]


class PipelineRunner:
    """One token at a time through the stages.  The ranks are in lockstep per token, so a context shift needs nothing from the
    runner: every rank calls its stage's kv_shift (Model.kv_shift) with the same arguments between the same two step() calls."""

    def __init__(self, stage, rank: int, world: int, dist=None, token_tensor=None, stream=None):
        self.stage, self.rank, self.world, self.dist = stage, rank, world, dist
        self.stream = stream      # the engine's stream as a torch stream: entered around every step (see the module docstring)
        self.tok = token_tensor   # int64[1] on the stage's device
        if world > 1 and dist is None:
            raise ValueError("world > 1 needs torch.distributed")

    @property
    def first(self) -> bool:
        return self.rank == 0

    @property
    def last(self) -> bool:
        return self.rank == self.world - 1

    def step(self, token: int, pos: int, sample=None) -> int | None:
        """Runs one token through the pipeline.  Returns the sampled token on rank 0 (None elsewhere / when world == 1 and no
        sampler is given).  `sample(logits_tensor) -> int64[1] tensor` runs on the last rank."""
        with _entered(self.stream):
            return self._step(token, pos, sample)

    def _step(self, token: int, pos: int, sample=None) -> int | None:
        st, d = self.stage, self.dist
        if self.world == 1:
            st.decode_async(token, pos)
            return None
        if not self.first:
            d.recv(st.hidden_in, src=self.rank - 1)
        st.decode_async(token, pos)
        if not self.last:
            d.send(st.hidden_out, dst=self.rank + 1)
        if self.last:
            # sample(logits) returns a 1-element device tensor (the engine's device argmax leaves it in place: no copy, no host sync)
            t = sample(st.logits).reshape(1)
            if t.data_ptr() != self.tok.data_ptr():
                self.tok.copy_(t)
            d.send(self.tok, dst=0)
        if self.first:
            # the returned token lands in device memory; the next step is ordered after it on the stream (no host round trip)
            d.recv(self.tok, src=self.world - 1)
            if not self.tok.is_cuda:
                return int(self.tok.item())     # CPU tensors (gloo tests): the value is already here
        return None


class RingRunner:
    """Several tokens in flight: prima's piped ring proper (src/llama.cpp:17825-18029, 18299-18387) with one independent sequence
    per stage, so that every GPU works in every time slot instead of one GPU at a time.

    world = N stages, S = N sequence slots.  In time slot t stage r runs its layers on sequence (t - r) mod N.  At the START of every
    slot each stage does ONE grouped exchange (ncclGroupStart/End through torch.distributed.batch_isend_irecv): it forwards the
    result of its previous slot (hidden state to stage r+1; the last stage returns the sampled token id to stage 0) and receives the
    input of this slot.  The exchange is a ring, grouped per stage, so it cannot deadlock, and nothing crosses the host: token ids
    and positions stay in device memory (pb200_step_seq_dev), the greedy sample is a device kernel (pb200_argmax_seq).

    The stage object provides: hidden_in / hidden_out (tensors aliasing the engine's buffers), token_in(seq) / token_out(seq)
    (int32[1] tensors: where a returned token lands on stage 0 / where the last stage leaves its sample), begin(seq, token, pos)
    (stage 0: first token of a sequence; other stages: position only) and run(seq) (one step of the slot, sampling included on the
    last stage), and kv_shift(seq, p0, p1, delta) where shift() is used.  prefill() also needs prefill_stage(..., seq=) and hidden_buf
    (as PrefillPipeline drives them) and, on the last stage, sample(seq) (the first token of the slot's logits -> token_out(seq)); copy()
    needs kv_copy(src, dst, p0, p1).  The same class drives CPU tensors over gloo in tests/test_pipeline_gloo.py and
    tests/test_ring_prompts_gloo.py."""

    def __init__(self, stage, rank: int, world: int, dist, stream=None):
        if world < 2 or dist is None:
            raise ValueError("RingRunner needs world >= 2 and torch.distributed")
        self.stage, self.rank, self.world, self.dist = stage, rank, world, dist
        self.stream = stream
        self.t = 0
        self.runs: dict[int, int] = {}                          # runs of each sequence on this rank so far
        self.shifts: dict[int, list[tuple[int, int, int, int]]] = {}
        self.copies: dict[int, list[tuple[int, int, int, int]]] = {}   # dst -> (at_step, src, p0, p1)

    def shift(self, seq: int, at_step: int, p0: int, p1: int, delta: int) -> None:
        """Context shift of sequence seq (prima forwards llama_kv_cache_seq_rm / seq_add down the ring, src/llama.cpp:17946, 18345):
        every rank applies stage.kv_shift(seq, p0, p1, delta) immediately before its own run number at_step (0-based) of seq, so
        the shift lands between the same two tokens of the sequence on every rank.  Stage r runs a given token of a sequence r time
        slots after stage 0, which is why the point is counted in runs of the sequence, not in time slots.  Call it with the same
        arguments on every rank, before that run."""
        if at_step < self.runs.get(seq, 0):
            raise ValueError(f"sequence {seq} has already run {self.runs.get(seq, 0)} steps on rank {self.rank}")
        self.shifts.setdefault(seq, []).append((at_step, p0, p1, delta))

    def copy(self, src: int, dst: int, at_step: int, p0: int = -1, p1: int = -1) -> None:
        """KV copy between sequences (prima's kv_seq_cp ring command, src/llama.cpp:17955): every rank applies
        stage.kv_copy(src, dst, p0, p1) immediately before its own run number at_step (0-based) of dst, like shift().  Every rank runs the
        sequences in the same order, so at that point src has also run the same number of steps on every rank.  Call it with the same
        arguments on every rank, before that run; positions are the caller's (the copy moves none)."""
        if at_step < self.runs.get(dst, 0):
            raise ValueError(f"sequence {dst} has already run {self.runs.get(dst, 0)} steps on rank {self.rank}")
        self.copies.setdefault(dst, []).append((at_step, src, p0, p1))

    def prefill(self, prompts, ubatch: int = 512) -> None:
        """Starts every sequence from a prompt: call it on every rank with the same prompts (one token list per sequence, world of them)
        before the first slots(), which then runs without first_tokens.  For each sequence s in turn the prompt goes through the stages in
        micro-batches into slot s (PrefillPipeline), the last stage samples the first token into token_out(s) (stage.sample(s)) and sends it
        to stage 0's token_in(s), and every stage sets the slot's position to len(prompts[s]) (begin(s, 0, len)).  On stage 0 the begin is
        ordered before the receive, so the received token overwrites the placeholder.  One send / recv pair per stage boundary and
        micro-batch, then one from the last stage to stage 0: each pair's sender finishes its part first, so the exchange cannot
        deadlock."""
        if self.t != 0:
            raise ValueError("prefill() starts the sequences: call it before the first slots()")
        if len(prompts) != self.world or not all(len(p) for p in prompts):
            raise ValueError(f"need one non-empty prompt per sequence ({self.world})")
        st, d, r, N = self.stage, self.dist, self.rank, self.world
        pipe = PrefillPipeline(st, r, N, d, ubatch=ubatch)
        with _entered(self.stream):
            for s, prompt in enumerate(prompts):
                n = len(prompt)
                pipe.run(prompt, n, 0, seq=s)
                st.begin(s, 0, n)
                if r == N - 1:
                    st.sample(s)
                    d.send(st.token_out(s), dst=0)
                elif r == 0:
                    d.recv(st.token_in(s), src=N - 1)

    def slots(self, n: int, first_tokens=None) -> None:
        """Runs time slots self.t .. self.t + n - 1 (the same n on every rank).  first_tokens[s] = (token, pos) seeds sequence s."""
        with _entered(self.stream):
            self._slots(n, first_tokens)

    def _slots(self, n: int, first_tokens=None) -> None:
        st, d, r, N = self.stage, self.dist, self.rank, self.world
        nxt, prv = (r + 1) % N, (r - 1) % N
        for _ in range(n):
            t = self.t
            a = t - r                      # this stage's slot index in its own sequence of work; < 0 while the pipeline fills
            ops = []
            if a - 1 >= 0:                 # forward the result of the previous slot
                sp = (a - 1) % N
                ops.append(d.P2POp(d.isend, st.token_out(sp) if r == N - 1 else st.hidden_out, nxt))
            if a >= 0:
                sq = a % N
                if r == 0:
                    if a >= N:
                        ops.append(d.P2POp(d.irecv, st.token_in(sq), prv))       # the token stage N-1 sampled for this sequence
                else:
                    ops.append(d.P2POp(d.irecv, st.hidden_in, prv))
            if ops:
                for w in d.batch_isend_irecv(ops):
                    w.wait()               # NCCL: orders the current stream after the exchange, does not block the host
            if a >= 0:
                sq = a % N
                if a < N and first_tokens is not None:
                    st.begin(sq, *first_tokens[sq])
                done = self.runs.get(sq, 0)
                for sh in [s for s in self.shifts.get(sq, ()) if s[0] == done]:
                    st.kv_shift(sq, *sh[1:])
                    self.shifts[sq].remove(sh)
                for cp in [c for c in self.copies.get(sq, ()) if c[0] == done]:
                    st.kv_copy(cp[1], sq, *cp[2:])
                    self.copies[sq].remove(cp)
                st.run(sq)
                self.runs[sq] = done + 1
            self.t += 1


class PrefillPipeline:
    """Prompt processing through the layer pipeline in micro-batches (the reference's n_ubatch = 512; prima ships the ubatch's hidden states
    from window to window, src/llama.cpp:17825-18029): stage r works on micro-batch j while stage r + 1 works on j - 1.

    The stage object provides prefill_stage(tokens | None, hidden_in | None, n, pos0) -> tensor [n, n_embd] (the stage's output hidden
    states, valid until its next call; pb200_prefill_stage enqueues on the engine stream and returns at once) and, on every stage but the
    first, a receive buffer hidden_buf [ubatch, n_embd].  One send / recv pair per stage boundary and micro-batch, in micro-batch order on
    both sides, so the exchange cannot deadlock; with NCCL everything is ordered on `stream`.  Every rank must call run() with the same
    token count.  The same class drives CPU tensors over gloo in tests/test_pipeline_gloo.py."""

    def __init__(self, stage, rank: int, world: int, dist, ubatch: int = 512, stream=None):
        if world < 2 or dist is None:
            raise ValueError("PrefillPipeline needs world >= 2 and torch.distributed")
        self.stage, self.rank, self.world, self.dist, self.ubatch, self.stream = stage, rank, world, dist, ubatch, stream

    def run(self, tokens, n_tokens: int, pos0: int = 0, seq: int = 0, outputs=None):
        """tokens: the prompt's token ids (read on rank 0 only).  seq: the sequence slot the prompt goes to; it is passed to the stage's
        prefill_stage as the keyword seq only when it is not 0, so a stage that only serves slot 0 keeps its four-argument method.
        outputs(j0, n): called on the last rank only, right after micro-batch [j0, j0 + n)'s prefill_stage and before the next one, while
        the stage's output hidden states still hold that micro-batch (Model.prompt_head reads them: the logits of any of its rows).  Returns
        the last micro-batch's output of this stage."""
        st, d, r = self.stage, self.dist, self.rank
        kw = {"seq": seq} if seq else {}
        out = None
        with _entered(self.stream):
            for j0 in range(0, n_tokens, self.ubatch):
                n = min(self.ubatch, n_tokens - j0)
                hin = None
                if r > 0:
                    hin = st.hidden_buf[:n]
                    d.recv(hin, src=r - 1)
                out = st.prefill_stage(tokens[j0:j0 + n] if r == 0 else None, hin, n, pos0 + j0, **kw)
                if outputs is not None and r == self.world - 1:
                    outputs(j0, n)
                if r < self.world - 1:
                    d.send(out, dst=r + 1)
        return out
