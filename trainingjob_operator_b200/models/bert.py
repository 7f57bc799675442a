"""BERT-base (masked-language-model pre-training) on the hand-written engine.

BASELINE.json's fault-injection config names "BERT-base DDP"; the reference operator contains no model code (SURVEY.md
§2.6), so this is one of the launched workers' benchmark workloads.  It is the real architecture -- not a relabelled
GPT-2: word + position + token-type embeddings followed by a LayerNorm, twelve POST-LayerNorm encoder layers with
bidirectional attention (``y = LN(x + Attn(x))``, ``x' = LN(y + MLP(y))``), and the MLM head (dense + GELU + LayerNorm,
decoder tied to the word embeddings plus its own bias) with the loss taken over the masked positions only (15 % of the
tokens; unmasked positions carry label -1).  GELU is the tanh form (``gelu_new``), which is what the GEMM epilogues fuse.

Everything runs on the kernels of ``ops/csrc``: wgmma GEMMs with fused bias / GELU / residual epilogues (forward and
input gradients; the residual epilogue of the dgrad GEMMs adds the skip connection's gradient), split-K weight-gradient
GEMMs into the flat fp32 gradient buffer, LayerNorm forward / backward (the backward also yields the bias gradient of the
linear layer in front of it), three-table embedding gather / scatter, softmax-cross-entropy with ignored labels, flat AdamW.
``BertReference`` is the plain fp32 PyTorch model on the same weights for the numerics tests.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Tuple

import torch
import torch.nn.functional as TF

from .engine import TransformerEngine
from .flat_params import FlatParams, ParamSpec

MASK_TOKEN = 103


@dataclass
class BertConfig:
    vocab_size: int = 30522
    n_layer: int = 12
    n_head: int = 12
    n_embd: int = 768
    block_size: int = 512            # max position embeddings
    type_vocab: int = 2
    name: str = "bert-base"

    @property
    def padded_vocab(self) -> int:
        return (self.vocab_size + 127) // 128 * 128

    @staticmethod
    def base() -> "BertConfig":
        return BertConfig()

    @staticmethod
    def tiny() -> "BertConfig":
        return BertConfig(vocab_size=1000, n_layer=2, n_head=4, n_embd=256, block_size=128, name="bert-tiny")


def bert_param_specs(cfg: BertConfig) -> List[ParamSpec]:
    """Matrices first (embeddings, per-layer weights, MLM transform), every 1-D parameter in one tail region."""
    C, L = cfg.n_embd, cfg.n_layer
    specs = [ParamSpec("wte", (cfg.padded_vocab, C), True), ParamSpec("wpe", (cfg.block_size, C), True),
             ParamSpec("wtt", (cfg.type_vocab, C), True)]
    for i in range(L):
        p = f"h{i}."
        specs += [ParamSpec(p + "qkv_w", (3 * C, C), True), ParamSpec(p + "proj_w", (C, C), True),
                  ParamSpec(p + "fc_w", (4 * C, C), True), ParamSpec(p + "fc2_w", (C, 4 * C), True)]
    specs.append(ParamSpec("mlm_w", (C, C), True))
    specs += [ParamSpec("emb_ln_w", (C,), False, "ones"), ParamSpec("emb_ln_b", (C,), False, "zeros")]
    for i in range(L):
        p = f"h{i}."
        specs += [ParamSpec(p + "qkv_b", (3 * C,), False, "zeros"), ParamSpec(p + "proj_b", (C,), False, "zeros"),
                  ParamSpec(p + "ln1_w", (C,), False, "ones"), ParamSpec(p + "ln1_b", (C,), False, "zeros"),
                  ParamSpec(p + "fc_b", (4 * C,), False, "zeros"), ParamSpec(p + "fc2_b", (C,), False, "zeros"),
                  ParamSpec(p + "ln2_w", (C,), False, "ones"), ParamSpec(p + "ln2_b", (C,), False, "zeros")]
    specs += [ParamSpec("mlm_b", (C,), False, "zeros"), ParamSpec("mlm_ln_w", (C,), False, "ones"),
              ParamSpec("mlm_ln_b", (C,), False, "zeros"), ParamSpec("dec_b", (cfg.padded_vocab,), False, "zeros")]
    return specs


def bert_flops_per_token(cfg: BertConfig, T: int) -> float:
    """fwd+bwd matmul FLOPs per token: 6 x (encoder weights + MLM transform + tied decoder) + bidirectional attention."""
    C, L = cfg.n_embd, cfg.n_layer
    dense = L * 12 * C * C + C * C + cfg.padded_vocab * C
    attn = L * 2 * T * C
    return 6.0 * dense + 6.0 * attn


class SyntheticMLM:
    """Synthetic masked-LM batches of the named shape in pinned host memory: tokens (15 % replaced by [MASK]), token
    types (two segments), labels (-1 except at the masked positions).  The number of masked positions is fixed so the
    loss scale is a constant of the captured graph."""

    def __init__(self, vocab: int, batch: int, seq: int, n_batches: int = 4, seed: int = 0, pin: bool = True):
        g = torch.Generator().manual_seed(seed)
        M = batch * seq
        self.n_masked = max(1, int(round(0.15 * M)))
        self.batches = []
        for _ in range(n_batches):
            tok = torch.randint(1000 if vocab > 2000 else 1, vocab, (M,), generator=g, dtype=torch.int64)
            typ = (torch.arange(M) % seq >= seq // 2).to(torch.int64)
            lab = torch.full((M,), -1, dtype=torch.int64)
            pos = torch.randperm(M, generator=g)[: self.n_masked]
            lab[pos] = tok[pos]
            tok = tok.clone()
            tok[pos] = MASK_TOKEN if vocab > MASK_TOKEN else 0
            ts = [tok, typ, lab]
            if pin and torch.cuda.is_available():
                ts = [t.pin_memory() for t in ts]
            self.batches.append(tuple(ts))
        self.i = 0
        self.bytes_per_step = 3 * M * 8

    def next(self):
        b = self.batches[self.i % len(self.batches)]
        self.i += 1
        return b


class BertEngine(TransformerEngine):
    """Explicit forward / backward / optimizer of BERT-base MLM pre-training for a fixed (B, T) micro-batch on one GPU,
    on ``TransformerEngine``.  Layer i's LN2 output, ``layers[i].ln2``, is the input of layer i + 1."""

    def __init__(self, cfg: BertConfig, batch_size: int, seq_len: int, device="cuda", seed: int = 0,
                 gemm_backend: str = "wgmma"):
        super().__init__(cfg, bert_param_specs(cfg), batch_size, seq_len, device, seed, gemm_backend, causal=False,
                         doc_mask=False)
        C, M = cfg.n_embd, self.M
        bf = dict(device=self.dev, dtype=torch.bfloat16)
        f32 = dict(device=self.dev, dtype=torch.float32)
        self.typ = torch.zeros(M, dtype=torch.int64, device=self.dev)
        self.tgt.fill_(-1)
        self.n_masked = max(1, int(round(0.15 * M)))
        self.e0 = torch.empty(M, C, **bf)                      # sum of the three embeddings
        self.x0 = torch.empty(M, C, **bf)                      # LN(e0): input of layer 0
        self.e_mean, self.e_rstd = torch.empty(M, **f32), torch.empty(M, **f32)
        self.mlm_pre = torch.empty(M, C, **bf)
        self.mlm_act = torch.empty(M, C, **bf)
        self.mlm_ln = torch.empty(M, C, **bf)
        self.m_mean, self.m_rstd = torch.empty(M, **f32), torch.empty(M, **f32)
        self.d_x = [torch.empty(M, C, **bf) for _ in range(3)]

    def input_tensors(self) -> List[torch.Tensor]:
        return [self.tok, self.typ, self.tgt]

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self) -> torch.Tensor:
        F, P = self.F, self.params
        F.embedding3_fwd(self.tok, self.typ, P.w16("wte"), P.w16("wpe"), P.w16("wtt"), self.e0, self.T)
        self.layernorm_fwd(self.e0, P.w16("emb_ln_w"), P.w16("emb_ln_b"), self.x0, self.e_mean, self.e_rstd)
        x = self.x0
        for i, lb in enumerate(self.layers):
            p = f"h{i}."
            self._linear(x, P.w16(p + "qkv_w"), lb.qkv, bias=P.w16(p + "qkv_b"))
            self._attention_fwd(lb)
            self._linear(lb.att_in, P.w16(p + "proj_w"), lb.res1, bias=P.w16(p + "proj_b"), residual=x)
            self.layernorm_fwd(lb.res1, P.w16(p + "ln1_w"), P.w16(p + "ln1_b"), lb.ln1, lb.ln1_mean, lb.ln1_rstd)   # y
            self._linear(lb.ln1, P.w16(p + "fc_w"), lb.fc_act, bias=P.w16(p + "fc_b"), gelu=True, aux=lb.fc_pre)
            self._linear(lb.fc_act, P.w16(p + "fc2_w"), lb.res2, bias=P.w16(p + "fc2_b"), residual=lb.ln1)
            self.layernorm_fwd(lb.res2, P.w16(p + "ln2_w"), P.w16(p + "ln2_b"), lb.ln2, lb.ln2_mean, lb.ln2_rstd)
            x = lb.ln2
        # MLM head: dense + GELU + LayerNorm, decoder tied to the word embeddings (+ its own bias)
        self._linear(x, P.w16("mlm_w"), self.mlm_act, bias=P.w16("mlm_b"), gelu=True, aux=self.mlm_pre)
        self.layernorm_fwd(self.mlm_act, P.w16("mlm_ln_w"), P.w16("mlm_ln_b"), self.mlm_ln, self.m_mean, self.m_rstd)
        self._linear(self.mlm_ln, P.w16("wte"), self.logits, bias=P.w16("dec_b"))
        return self._loss(self.n_masked)

    # ------------------------------------------------------------------ backward segments
    @torch.no_grad()
    def _bwd_head(self) -> None:
        F, P = self.F, self.params
        dlogits = self.logits
        x_last = self.layers[-1].ln2 if self.layers else self.x0
        d_t, d_g, d_u = self.d_x
        F.colsum(dlogits, P.grad("dec_b"))
        self._dgrad(dlogits, P.w16("wte"), d_t)
        self._wgrad(dlogits, self.mlm_ln, P.grad("wte"))
        self.layernorm_bwd(d_t, self.mlm_act, P.w16("mlm_ln_w"), self.m_mean, self.m_rstd, d_g, P.grad("mlm_ln_w"),
                           P.grad("mlm_ln_b"))
        F.gelu_bwd(self.mlm_pre, d_g, d_u)
        F.colsum(d_u, P.grad("mlm_b"))
        self._wgrad(d_u, x_last, P.grad("mlm_w"))
        self._dgrad(d_u, P.w16("mlm_w"), d_t)                # (the weight gradients above read dlogits, mlm_ln, d_u, x_last:
        self._d_cur = d_t                                    #  none of them is written again before the next layer's join)
        if self.segment_join:
            self._join_wgrads()

    @torch.no_grad()
    def _bwd_layer(self, i: int) -> None:
        F, P = self.F, self.params
        lb = self.layers[i]
        p = f"h{i}."
        x_in = self.layers[i - 1].ln2 if i > 0 else self.x0
        self._join_wgrads()                                  # last segment's weight gradients still read these buffers
        free = [t for t in self.d_x if t is not self._d_cur]
        d_r, d_y = free
        # x_{l+1} = LN2(y + MLP(y))
        self.layernorm_bwd(self._d_cur, lb.res2, P.w16(p + "ln2_w"), lb.ln2_mean, lb.ln2_rstd, d_r,
                           P.grad(p + "ln2_w"), P.grad(p + "ln2_b"), dxsum=P.grad(p + "fc2_b"))
        e_fc2 = self._wgrad(d_r, lb.fc_act, P.grad(p + "fc2_w"))
        self._dgrad(d_r, P.w16(p + "fc2_w"), self.d_fc, dgelu_aux=lb.fc_pre, colsum=P.grad(p + "fc_b"))
        self._wgrad(self.d_fc, lb.ln1, P.grad(p + "fc_w"))
        self._dgrad(self.d_fc, P.w16(p + "fc_w"), d_y, residual=d_r)            # + the skip connection's gradient
        # y = LN1(x + Attn(x))
        d_r1 = self._d_cur                                                      # its content is no longer needed
        self.layernorm_bwd(d_y, lb.res1, P.w16(p + "ln1_w"), lb.ln1_mean, lb.ln1_rstd, d_r1, P.grad(p + "ln1_w"),
                           P.grad(p + "ln1_b"), dxsum=P.grad(p + "proj_b"))
        self._wgrad(d_r1, lb.att_in, P.grad(p + "proj_w"))
        self._dgrad(d_r1, P.w16(p + "proj_w"), self.d_att)
        self._attention_bwd(lb, self.d_att, self.d_qkv, P.grad(p + "qkv_b"))
        self._wgrad(self.d_qkv, x_in, P.grad(p + "qkv_w"))
        if e_fc2 is not None:
            torch.cuda.current_stream().wait_event(e_fc2)     # d_r is the buffer the fc2 weight gradient read
        self._dgrad(self.d_qkv, P.w16(p + "qkv_w"), d_r, residual=d_r1)
        self._d_cur = d_r
        if self.segment_join:
            self._join_wgrads()

    @torch.no_grad()
    def _bwd_tail(self) -> None:
        F, P = self.F, self.params
        # layer 0's weight-gradient GEMMs may still read the buffer d_e is about to occupy (found by the late-stream model
        # of tests/kernel_emulation.py: h0.proj_w came out wrong with AITJ_WGRAD_STREAM=1)
        self._join_wgrads()
        d_e = next(t for t in self.d_x if t is not self._d_cur)
        self.layernorm_bwd(self._d_cur, self.e0, P.w16("emb_ln_w"), self.e_mean, self.e_rstd, d_e, P.grad("emb_ln_w"),
                           P.grad("emb_ln_b"))
        F.embedding3_bwd(self.tok, self.typ, d_e, P.grad("wte"), P.grad("wpe"), P.grad("wtt"), self.T)
        P.push_small_grads()
        self._join_wgrads()

    # ------------------------------------------------------------------ buckets (for DDP)
    def grad_buckets(self) -> List[Tuple[str, int, int]]:
        P = self.params
        out = []
        for i in range(self.cfg.n_layer - 1, -1, -1):
            out.append((f"h{i}",) + P.range_of(f"h{i}.qkv_w", f"h{i}.fc2_w"))
        out.append(("emb",) + P.range_of("wte", "wtt"))
        out.append(("small",) + P.range_of("mlm_w", "dec_b"))
        return out


# ------------------------------------------------------------------------------------ reference
class BertReference(torch.nn.Module):
    """Plain PyTorch BERT-base MLM (fp32) reading the engine's master weights; used for numerics checks."""

    def __init__(self, cfg: BertConfig, params: FlatParams):
        super().__init__()
        self.cfg = cfg
        self.w = torch.nn.ParameterDict({s.name.replace(".", "_"): torch.nn.Parameter(params.w32(s.name).clone())
                                         for s in params.specs})

    def p(self, name: str) -> torch.Tensor:
        return self.w[name.replace(".", "_")]

    def forward(self, tok: torch.Tensor, typ: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        cfg = self.cfg
        B, T = tok.shape
        C, H = cfg.n_embd, cfg.n_head
        x = self.p("wte")[tok] + self.p("wpe")[:T] + self.p("wtt")[typ]
        x = TF.layer_norm(x, (C,), self.p("emb_ln_w"), self.p("emb_ln_b"))
        for i in range(cfg.n_layer):
            q = f"h{i}."
            qkv = x @ self.p(q + "qkv_w").t() + self.p(q + "qkv_b")
            qh, kh, vh = [t.view(B, T, H, C // H).transpose(1, 2) for t in qkv.split(C, dim=-1)]
            a = TF.scaled_dot_product_attention(qh, kh, vh).transpose(1, 2).reshape(B, T, C)
            y = TF.layer_norm(x + a @ self.p(q + "proj_w").t() + self.p(q + "proj_b"), (C,), self.p(q + "ln1_w"),
                              self.p(q + "ln1_b"))
            h = TF.gelu(y @ self.p(q + "fc_w").t() + self.p(q + "fc_b"), approximate="tanh")
            x = TF.layer_norm(y + h @ self.p(q + "fc2_w").t() + self.p(q + "fc2_b"), (C,), self.p(q + "ln2_w"),
                              self.p(q + "ln2_b"))
        t = TF.gelu(x @ self.p("mlm_w").t() + self.p("mlm_b"), approximate="tanh")
        t = TF.layer_norm(t, (C,), self.p("mlm_ln_w"), self.p("mlm_ln_b"))
        logits = t @ self.p("wte")[:cfg.vocab_size].t() + self.p("dec_b")[:cfg.vocab_size]
        return TF.cross_entropy(logits.view(B * T, -1), labels.view(-1), ignore_index=-1)
