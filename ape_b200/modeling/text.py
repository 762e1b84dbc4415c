"""EVA02-CLIP text tower (SURVEY.md §8(f) row 1): `model_language.forward_text` for free-text prompts.

Mirror of ape/modeling/text/clip_wrapper_eva02.py:16-158 (`EVA02CLIP`: tokenize -> text transformer -> features of the
end-of-text token and of every token) and of the `TextTransformer` it wraps (ape/modeling/text/eva02_clip/transformer.py:
642-737, blocks :443-483: pre-LayerNorm residual blocks, nn.MultiheadAttention with the causal mask of :714-720, GELU MLP x4):
same constructor arguments, same parameter names (`net.text.token_embedding`, `…positional_embedding`,
`…transformer.resblocks.{i}.{ln_1,attn.in_proj_weight,attn.in_proj_bias,attn.out_proj,ln_2,mlp.c_fc,mlp.c_proj}`,
`…ln_final`, `…text_projection`, `net.logit_scale`), so the text half of an EVA02-CLIP checkpoint loads by name.

Engine path (CUDA, fp16 / bf16 — the reference runs this tower in fp16, clip_wrapper_eva02.py:31-43): every linear is a
wgmma GEMM, the attention is the repo's flash-attention kernel with the causal mask and the 77-token prompts packed at a
row stride of 80, LayerNorms are the repo's row kernels, the residual stream is fp32.  EVA02-CLIP-bigE-14-plus: width 1280,
20 heads x 64, 32 layers, 97 GFLOP per prompt — for uncached `--text-prompt` lists it dwarfs the vision path."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops


class _MLP(nn.Sequential):
    def __init__(self, width, hidden):
        super().__init__()
        self.add_module("c_fc", nn.Linear(width, hidden))
        self.add_module("gelu", nn.GELU())
        self.add_module("c_proj", nn.Linear(hidden, width))


class ResidualAttentionBlock(nn.Module):
    def __init__(self, d_model, n_head, mlp_ratio=4.0):
        super().__init__()
        self.ln_1 = nn.LayerNorm(d_model)
        self.attn = nn.MultiheadAttention(d_model, n_head)
        self.ln_2 = nn.LayerNorm(d_model)
        self.mlp = _MLP(d_model, int(d_model * mlp_ratio))

    def forward(self, x, attn_mask=None):  # x [L, N, D] (the reference's LND layout), literal path
        h = self.ln_1(x)
        x = x + self.attn(h, h, h, need_weights=False, attn_mask=attn_mask)[0]
        return x + self.mlp(self.ln_2(x))


class Transformer(nn.Module):
    def __init__(self, width, layers, heads, mlp_ratio=4.0):
        super().__init__()
        self.width, self.layers = width, layers
        self.resblocks = nn.ModuleList([ResidualAttentionBlock(width, heads, mlp_ratio) for _ in range(layers)])

    def forward(self, x, attn_mask=None):
        for r in self.resblocks:
            x = r(x, attn_mask=attn_mask)
        return x


class TextTransformer(nn.Module):
    def __init__(self, context_length=77, vocab_size=49408, width=512, heads=8, layers=12, output_dim=512, **_ignored):
        super().__init__()
        self.context_length, self.vocab_size, self.width, self.output_dim, self.heads = context_length, vocab_size, width, output_dim, heads
        self.token_embedding = nn.Embedding(vocab_size, width)
        self.positional_embedding = nn.Parameter(torch.empty(context_length, width))
        self.transformer = Transformer(width, layers, heads)
        self.ln_final = nn.LayerNorm(width)
        self.text_projection = nn.Parameter(torch.empty(width, output_dim))
        mask = torch.full((context_length, context_length), float("-inf")).triu_(1)
        self.register_buffer("attn_mask", mask, persistent=False)
        nn.init.normal_(self.token_embedding.weight, std=0.02)
        nn.init.normal_(self.positional_embedding, std=0.01)
        nn.init.normal_(self.text_projection, std=width ** -0.5)

    # ---- literal path (fp32, any device): eva02_clip/transformer.py:722-737 + clip_wrapper_eva02.py:131-150 ----
    def encode(self, text):
        """text int64 [N, ctx] -> (features of the end-of-text token [N, out], features of every token [N, ctx, out])."""
        if text.is_cuda and self.text_projection.is_cuda and self.engine_dtype is not None and self.width // self.heads == 64:
            return self._encode_engine(text, self.engine_dtype)
        x = self.token_embedding(text) + self.positional_embedding
        x = self.transformer(x.permute(1, 0, 2), attn_mask=self.attn_mask).permute(1, 0, 2)
        x = self.ln_final(x)
        xx = x @ self.text_projection
        return x[torch.arange(x.shape[0]), text.argmax(dim=-1)] @ self.text_projection, xx

    engine_dtype = torch.float16  # None: literal path on CUDA as well

    # ---- engine path ---------------------------------------------------------------------------------------------
    def _encode_engine(self, text, dt):
        N, L = text.shape
        D, H = self.width, self.heads
        stride = (L + 7) // 8 * 8          # 77-token prompts packed at 80 rows: 16-byte aligned 16-bit rows of a sequence start
        n_tile = (L + 127) // 128 * 128    # attention tile
        M = N * stride
        x = (self.token_embedding(text) + self.positional_embedding).float()           # [N, L, D] fp32 residual stream
        xs = torch.zeros((N, stride, D), dtype=torch.float32, device=text.device)
        xs[:, :L] = x
        x = xs.view(M, D)
        for blk in self.transformer.resblocks:
            h = ops.layernorm_module(blk.ln_1, x, out_dtype=dt)
            w_in, b_in = ops.cached(blk.attn, "_ape_in", dt, (blk.attn.in_proj_weight._version, blk.attn.in_proj_weight.data_ptr()),
                                    lambda: (blk.attn.in_proj_weight.detach().to(dt).contiguous(),
                                             blk.attn.in_proj_bias.detach().float().contiguous()))
            qkv = ops.linear_tc(h, w_in, b_in)                                          # [M, 3D]: q | k | v, heads contiguous
            o = ops.attention_qkv(qkv, N, n_tile, H, 64, 0.125, n_valid=L, seq_stride=stride, causal=True)
            # rows between L and the stride hold stale values; they never mix with real rows (row-wise ops + masked keys)
            x = ops.linear_module_tc(blk.attn.out_proj, o, residual=x, out_dtype=torch.float32)
            h = ops.layernorm_module(blk.ln_2, x, out_dtype=dt)
            u = ops.linear_module_tc(blk.mlp.c_fc, h, act="gelu")
            x = ops.linear_module_tc(blk.mlp.c_proj, u, residual=x, out_dtype=torch.float32)
        xn = ops.layernorm_module(self.ln_final, x, out_dtype=dt)                       # [M, D]
        wp = ops.cached(self, "_ape_proj", dt, (self.text_projection._version, self.text_projection.data_ptr()),
                        lambda: self.text_projection.detach().t().to(dt).contiguous())
        xx = ops.linear_tc(xn, wp, None, out_dtype=torch.float32).view(N, stride, -1)[:, :L]
        eot = text.argmax(dim=-1)
        return xx[torch.arange(N, device=text.device), eot], xx


class _CLIPText(nn.Module):
    """The part of the EVA02-CLIP `CustomCLIP` object the wrapper keeps (`self.net.text`, `self.net.logit_scale`)."""

    def __init__(self, text_cfg, embed_dim):
        super().__init__()
        self.text = TextTransformer(output_dim=embed_dim, **text_cfg)
        self.logit_scale = nn.Parameter(torch.ones([]) * 2.6592600)  # log(1 / 0.07)


class EVA02CLIP(nn.Module):
    """clip_wrapper_eva02.py:16-158.  `tokenizer`: callable list[str] -> int64 [N, ctx] (the reference's
    `eva02_clip.tokenizer.tokenize`, whose BPE vocabulary ships with the reference package); pre-tokenised tensors are
    accepted directly.  Returns the reference's dict: last_hidden_state_eot, last_hidden_state, attention_mask, end_token_idx."""

    CONFIGS = {"EVA02-CLIP-bigE-14-plus": dict(embed_dim=1024, text_cfg=dict(context_length=77, vocab_size=49408, width=1280, heads=20, layers=32))}

    def __init__(self, clip_model="EVA02-CLIP-bigE-14-plus", cache_dir=None, dtype="float16", max_batch_size=2560, tokenizer=None,
                 text_cfg=None, embed_dim=None):
        super().__init__()
        cfg = self.CONFIGS.get(clip_model, {})
        self.net = _CLIPText(text_cfg or cfg["text_cfg"], embed_dim or cfg["embed_dim"])
        self.max_batch_size = max_batch_size
        self.tokenizer = tokenizer
        self.dtype = dtype
        self.net.text.engine_dtype = {"float16": torch.float16, "bfloat16": torch.bfloat16, "float32": None}[dtype]
        self.text_list_to_feature = {}
        self.register_buffer("unused_tensor", torch.zeros(1), False)
        self.eval()

    @property
    def device(self):
        return self.unused_tensor.device

    def _tokenize(self, text_list):
        if torch.is_tensor(text_list):
            return text_list
        tok = self.tokenizer
        if tok is None:
            try:
                from ape.modeling.text.eva02_clip import tokenizer as _t  # the reference package, when installed

                tok = _t.tokenize
            except Exception as e:  # noqa: BLE001
                raise RuntimeError("ape_b200.EVA02CLIP needs a tokenizer (the reference's eva02_clip.tokenizer.tokenize) "
                                   "or pre-tokenised int64 [N, 77] input") from e
        return tok(list(text_list))

    @torch.no_grad()
    def forward_text(self, text_list, cache=False):
        key = None if torch.is_tensor(text_list) else tuple(text_list)
        if cache and key is not None and key in self.text_list_to_feature:
            return self.text_list_to_feature[key]
        tokens = self._tokenize(text_list).to(self.device)
        xs, xxs = [], []
        for i in range(0, len(tokens), self.max_batch_size):      # (:94-112) chunks bound the activation memory
            x, xx = self.net.text.encode(tokens[i:i + self.max_batch_size])
            xs.append(x)
            xxs.append(xx)
        x, xx = torch.cat(xs), torch.cat(xxs)
        end = tokens.argmax(dim=-1)
        mask = (torch.arange(tokens.shape[1], device=tokens.device)[None] <= end[:, None]).to(end.dtype)
        ret = {"end_token_idx": end, "attention_mask": mask, "last_hidden_state": xx, "last_hidden_state_eot": x}
        if cache and key is not None:
            self.text_list_to_feature[key] = ret
        return ret
