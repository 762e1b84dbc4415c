"""EVA02-CLIP and EVA01-CLIP text towers (SURVEY.md §8(f) row 1): `model_language.forward_text` for free-text prompts.

Mirror of ape/modeling/text/clip_wrapper_eva02.py:16-158 (`EVA02CLIP`: tokenize -> text transformer -> features of the
end-of-text token and of every token) and of the `TextTransformer` it wraps (ape/modeling/text/eva02_clip/transformer.py:
642-737, blocks :443-483: pre-LayerNorm residual blocks, nn.MultiheadAttention with the causal mask of :714-720, GELU MLP x4):
same constructor arguments, same parameter names (`net.text.token_embedding`, `…positional_embedding`,
`…transformer.resblocks.{i}.{ln_1,attn.in_proj_weight,attn.in_proj_bias,attn.out_proj,ln_2,mlp.c_fc,mlp.c_proj}`,
`…ln_final`, `…text_projection`, `net.logit_scale`), so the text half of an EVA02-CLIP checkpoint loads by name.

Engine path (CUDA, fp16 / bf16 — the reference runs this tower in fp16, clip_wrapper_eva02.py:31-43): every linear is a
wgmma GEMM, the attention is the repo's flash-attention kernel with the causal mask and the 77-token prompts packed at a
row stride of 80, LayerNorms are the repo's row kernels, the residual stream is fp32.  EVA02-CLIP-bigE-14-plus: width 1280,
20 heads x 64, 32 layers, 97 GFLOP per prompt — for uncached `--text-prompt` lists it dwarfs the vision path.

EVA01-CLIP (ape/modeling/text/clip_wrapper_eva01.py, eva01_clip/eva_model.py:126-265: the language model of APE-L_A / L_B /
L_C) has the same blocks and parameter names (width 768, 12 heads x 64, 12 layers, GELU, 768 -> 1024 projection), so the
same TextTransformer and engine path run it; only the wrapper's parameter layout and weight loading differ.

Length-packed mode (`pack_prompts=True`, engine path only): only the row of the end-of-text token is read downstream and the
attention is causal, so the positions after that token are work nobody uses.  The mode drops them: the prompts' real tokens
are laid back to back in tiles of 128 rows (`pack_layout`), the attention masks across prompts inside a tile
(ape_attn_fwd_seg), and a class name costs its 3 to 8 tokens instead of 80 rows."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops


PACK_TILE = 128  # rows of an attention tile: a packed prompt never straddles one


def pack_layout(lengths, context_length=77):
    """Row layout of length-packed prompts.  lengths[i]: tokens of prompt i up to and including its end-of-text token.

    Next-fit in input order: prompt i goes behind prompt i - 1 when the current tile of 128 rows still has lengths[i] free
    rows, otherwise it opens the next tile and the rows left over stay pad rows.  So prompts keep their order inside and
    across tiles, no prompt straddles a tile, and the layout depends on nothing but `lengths`.  Returns numpy arrays:
      tiles      T; the layout has M = 128 T rows
      src   [M]  int32  index into the flattened [N, context_length] token matrix of the row's token; 0 on pad rows
      pos   [M]  int32  position of the row inside its prompt; -1 on pad rows
      seg_start [M] int32  row, within its tile, where the row's prompt starts; a pad row: its own row within the tile
      eot_row [N] int64 row of each prompt's end-of-text token
      rows  [sum(lengths)] int64  the real rows in (prompt, position) order, i.e. the rows `src[rows]` enumerates."""
    lens = np.asarray(lengths, dtype=np.int64).reshape(-1)
    if lens.size == 0 or lens.min() < 1 or lens.max() > min(PACK_TILE, context_length):
        raise ValueError(f"pack_layout: prompt lengths must lie in [1, {min(PACK_TILE, context_length)}] and there must be a prompt")
    tile, start = np.empty_like(lens), np.empty_like(lens)
    t = used = 0
    for i, n in enumerate(lens.tolist()):
        if used + n > PACK_TILE:
            t, used = t + 1, 0
        tile[i], start[i] = t, used
        used += n
    M = (t + 1) * PACK_TILE
    row0 = tile * PACK_TILE + start
    prompt = np.repeat(np.arange(lens.size), lens)
    p = np.arange(prompt.size) - np.repeat(np.cumsum(lens) - lens, lens)
    rows = row0[prompt] + p
    src, pos = np.zeros(M, np.int32), np.full(M, -1, np.int32)
    seg_start = (np.arange(M) % PACK_TILE).astype(np.int32)
    src[rows], pos[rows], seg_start[rows] = prompt * context_length + p, p, start[prompt]
    return {"tiles": t + 1, "src": src, "pos": pos, "seg_start": seg_start, "eot_row": row0 + lens - 1, "rows": rows}


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
    def encode(self, text, lengths=None, need_hidden=True):
        """text int64 [N, ctx] -> (features of the end-of-text token [N, out], features of every token [N, ctx, out]).
        `lengths` (host ints, argmax(text) + 1 per prompt; read from the device when None) and `need_hidden` only matter to the
        engine path with `pack_prompts`: need_hidden=False returns None for the features of every token."""
        if text.is_cuda and self.text_projection.is_cuda and self.engine_dtype is not None and self.width // self.heads == 64:
            if self.pack_prompts:
                return self._encode_engine_packed(text, self.engine_dtype, lengths, need_hidden)
            return self._encode_engine(text, self.engine_dtype)
        x = self.token_embedding(text) + self.positional_embedding
        x = self.transformer(x.permute(1, 0, 2), attn_mask=self.attn_mask).permute(1, 0, 2)
        x = self.ln_final(x)
        xx = x @ self.text_projection
        return x[torch.arange(x.shape[0]), text.argmax(dim=-1)] @ self.text_projection, xx

    engine_dtype = torch.float16  # None: literal path on CUDA as well
    # True: the engine path runs the prompts length-packed (module docstring).  Features of every token are then zeros after
    # the end-of-text token, where the padded layout returns what it computes from the pad tokens; nothing else differs
    # beyond 16-bit rounding of the attention.  A chunk whose packed layout would have no fewer rows than the padded one (long
    # prompts, or a single prompt) runs padded.  Off by default; measured on an H100 in DESIGN.md §5: many times faster for
    # lists of names and phrases, level for a handful of expressions and for prompts that fill the context.
    pack_prompts = False

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
        x = self._engine_blocks(xs.view(M, D), dt, lambda qkv: ops.attention_qkv(qkv, N, n_tile, H, 64, 0.125, n_valid=L,
                                                                                   seq_stride=stride, causal=True))
        xx = self._engine_project(x, dt).view(N, stride, -1)[:, :L]
        eot = text.argmax(dim=-1)
        return xx[torch.arange(N, device=text.device), eot], xx

    def _engine_blocks(self, x, dt, attend):
        """The residual blocks over x fp32 [M, D]; attend: qkv [M, 3D] -> attention output [M, D]."""
        for blk in self.transformer.resblocks:
            h = ops.layernorm_module(blk.ln_1, x, out_dtype=dt)
            w_in, b_in = ops.cached(blk.attn, "_ape_in", dt, (blk.attn.in_proj_weight._version, blk.attn.in_proj_weight.data_ptr()),
                                    lambda: (blk.attn.in_proj_weight.detach().to(dt).contiguous(),
                                             blk.attn.in_proj_bias.detach().float().contiguous()))
            qkv = ops.linear_tc(h, w_in, b_in)                                          # [M, 3D]: q | k | v, heads contiguous
            o = attend(qkv)
            # rows that hold no token (between L and the stride; pad rows of a packed tile) carry values of their own; they
            # never mix with real rows (row-wise ops + masked keys)
            x = ops.linear_module_tc(blk.attn.out_proj, o, residual=x, out_dtype=torch.float32)
            h = ops.layernorm_module(blk.ln_2, x, out_dtype=dt)
            u = ops.linear_module_tc(blk.mlp.c_fc, h, act="gelu")
            x = ops.linear_module_tc(blk.mlp.c_proj, u, residual=x, out_dtype=torch.float32)
        return x

    def _engine_project(self, x, dt):
        """ln_final and the text projection over the rows of x fp32 [M, D] -> fp32 [M, out]."""
        xn = ops.layernorm_module(self.ln_final, x, out_dtype=dt)
        wp = ops.cached(self, "_ape_proj", dt, (self.text_projection._version, self.text_projection.data_ptr()),
                        lambda: self.text_projection.detach().t().to(dt).contiguous())
        return ops.linear_tc(xn, wp, None, out_dtype=torch.float32)

    def _encode_engine_packed(self, text, dt, lengths, need_hidden):
        N, L = text.shape
        dev = text.device
        if lengths is None:
            lengths = (text.argmax(dim=-1) + 1).tolist()                                # the one device-to-host copy
        lay = pack_layout(lengths, L)
        if lay["tiles"] * PACK_TILE >= N * ((L + 7) // 8 * 8):
            # prompts so long that few share a tile (one of 77 tokens fills 128 rows against 80 padded): the padded layout
            # has fewer rows, so it runs; its features after the end-of-text token are zeroed to keep the mode's contract
            eot, xx = self._encode_engine(text, dt)
            if not need_hidden:
                return eot, None
            keep = torch.arange(L, device=dev)[None] < torch.as_tensor(lengths, device=dev)[:, None]
            return eot, xx * keep[..., None]
        src, pos, seg = torch.from_numpy(np.stack([lay["src"], lay["pos"], lay["seg_start"]])).to(dev)
        eot_row = torch.from_numpy(lay["eot_row"]).to(dev)
        tok = torch.where(pos >= 0, text.reshape(-1)[src.long()], 0).to(torch.int32)
        x = ops.text_embed_packed(self.token_embedding.weight.detach(), self.positional_embedding.detach(), tok, pos)
        x = self._engine_blocks(x, dt, lambda qkv: ops.attention_qkv(qkv, lay["tiles"], PACK_TILE, self.heads, 64, 0.125,
                                                                     causal=True, seg_start=seg))
        if not need_hidden:                                                             # N rows instead of 128 T
            return self._engine_project(ops.rows_gather(x, eot_row), dt), None
        proj = self._engine_project(x, dt)
        rows = torch.from_numpy(lay["rows"]).to(dev)
        xx = torch.zeros((N * L, proj.shape[1]), dtype=proj.dtype, device=dev)
        xx[src[rows].long()] = proj[rows]
        return ops.rows_gather(proj, eot_row), xx.view(N, L, -1)


class _CLIPText(nn.Module):
    """The part of the EVA02-CLIP `CustomCLIP` object the wrapper keeps (`self.net.text`, `self.net.logit_scale`)."""

    def __init__(self, text_cfg, embed_dim):
        super().__init__()
        self.text = TextTransformer(output_dim=embed_dim, **text_cfg)
        self.logit_scale = nn.Parameter(torch.ones([]) * 2.6592600)  # log(1 / 0.07)


class _EVA01Text(nn.Module):
    """The part of the EVA01-CLIP `EVA_CLIP` object the wrapper keeps (`self.net.text`, with `logit_scale` inside the text
    tower: eva01_clip/eva_model.py:193-219).  The blocks' `ln_attn` / `mlp.ln` are parameter-free identities there."""

    def __init__(self, text_cfg, embed_dim):
        super().__init__()
        self.text = TextTransformer(output_dim=embed_dim, **text_cfg)
        self.text.logit_scale = nn.Parameter(torch.ones([]) * 2.6592600)  # log(1 / 0.07)


_DTYPES = {"float16": torch.float16, "bfloat16": torch.bfloat16, "float32": None}


class _CLIPTextWrapper(nn.Module):
    """What the EVA01 / EVA02 wrappers share: tokenise -> text tower in chunks of max_batch_size -> the reference's
    `forward_text` dict (last_hidden_state_eot, last_hidden_state, attention_mask, end_token_idx), optionally cached per list.
    `tokenizer`: callable list[str] -> int64 [N, ctx]; pre-tokenised tensors are accepted directly.  `dtype` float16 /
    bfloat16 runs the tower's engine path on CUDA, float32 its literal path.

    `pack_prompts` (default False; also settable later): the engine path runs the prompts length-packed, so a prompt costs
    its own tokens and not the 77 positions of the context (TextTransformer.pack_prompts).  Turn it on for lists of names or
    phrases.  `last_hidden_state` then holds zeros after each prompt's end-of-text token, positions `attention_mask` marks
    invalid anyway; `forward_text(..., need_hidden=False)` skips that tensor (None) and reads out the end-of-text rows only."""

    @property
    def pack_prompts(self):
        return self.net.text.pack_prompts

    @pack_prompts.setter
    def pack_prompts(self, on):
        self.net.text.pack_prompts = bool(on)

    def _setup(self, dtype, max_batch_size, tokenizer, pack_prompts=False):
        self.pack_prompts = pack_prompts
        self.max_batch_size = max_batch_size
        self.tokenizer = tokenizer
        self.dtype = dtype
        self.net.text.engine_dtype = _DTYPES[dtype]
        self.text_list_to_feature = {}
        self.register_buffer("unused_tensor", torch.zeros(1), False)
        self.eval()

    @property
    def device(self):
        return self.unused_tensor.device

    def _default_tokenizer(self):
        raise NotImplementedError

    def _tokenize(self, text_list):
        if torch.is_tensor(text_list):
            return text_list
        tok = self.tokenizer or self._default_tokenizer()
        return tok(list(text_list))

    @torch.no_grad()
    def forward_text(self, text_list, cache=False, need_hidden=True):
        key = None if torch.is_tensor(text_list) else tuple(text_list)
        if cache and key is not None and key in self.text_list_to_feature:
            ret = self.text_list_to_feature[key]
            if ret["last_hidden_state"] is not None or not need_hidden:
                return ret
        tokens = self._tokenize(text_list).to(self.device)
        end = tokens.argmax(dim=-1)
        lengths = (end + 1).tolist() if self.pack_prompts and tokens.is_cuda else None  # one copy to the host per call
        xs, xxs = [], []
        for i in range(0, len(tokens), self.max_batch_size):      # (:94-112) chunks bound the activation memory
            x, xx = self.net.text.encode(tokens[i:i + self.max_batch_size],
                                         lengths and lengths[i:i + self.max_batch_size], need_hidden)
            xs.append(x)
            xxs.append(xx)
        x, xx = torch.cat(xs), (None if xxs[0] is None else torch.cat(xxs))
        mask = (torch.arange(tokens.shape[1], device=tokens.device)[None] <= end[:, None]).to(end.dtype)
        ret = {"end_token_idx": end, "attention_mask": mask, "last_hidden_state": xx, "last_hidden_state_eot": x}
        if cache and key is not None:
            self.text_list_to_feature[key] = ret
        return ret


class EVA02CLIP(_CLIPTextWrapper):
    """clip_wrapper_eva02.py:16-158.  `tokenizer`: the reference's `eva02_clip.tokenizer.tokenize`, whose BPE vocabulary ships
    with the reference package, by default."""

    CONFIGS = {"EVA02-CLIP-bigE-14-plus": dict(embed_dim=1024, text_cfg=dict(context_length=77, vocab_size=49408, width=1280, heads=20, layers=32))}

    def __init__(self, clip_model="EVA02-CLIP-bigE-14-plus", cache_dir=None, dtype="float16", max_batch_size=2560, tokenizer=None,
                 text_cfg=None, embed_dim=None, pack_prompts=False):
        super().__init__()
        cfg = self.CONFIGS.get(clip_model, {})
        self.net = _CLIPText(text_cfg or cfg["text_cfg"], embed_dim or cfg["embed_dim"])
        self._setup(dtype, max_batch_size, tokenizer, pack_prompts)

    def _default_tokenizer(self):
        try:
            from ape.modeling.text.eva02_clip import tokenizer as _t  # the reference package, when installed

            return _t.tokenize
        except Exception as e:  # noqa: BLE001
            raise RuntimeError("ape_b200.EVA02CLIP needs a tokenizer (the reference's eva02_clip.tokenizer.tokenize) "
                               "or pre-tokenised int64 [N, 77] input") from e


def load_eva01_text_state_dict(path):
    """The text half of an EVA01-CLIP checkpoint, read as eva01_clip/eva_clip.py:load_state_dict reads it: the state dict is
    under `model`, `module` or `state_dict` (first found) or is the file's dict itself, a leading `module.` is stripped, then
    the `text.*` entries are kept (without the prefix) and the vision tower's `visual.*` ones dropped."""
    ckpt = torch.load(path, map_location="cpu")
    sd = ckpt
    for mk in ("model", "module", "state_dict"):
        if isinstance(ckpt, dict) and mk in ckpt:
            sd = ckpt[mk]
            break
    if not isinstance(sd, dict) or not sd:
        raise ValueError(f"ape_b200.EVA01CLIP: {path} holds no state dict")
    if next(iter(sd)).startswith("module"):
        sd = {k[7:]: v for k, v in sd.items()}
    return {k[5:]: v for k, v in sd.items() if k.startswith("text.")}


class EVA01CLIP(_CLIPTextWrapper):
    """clip_wrapper_eva01.py:10-146: the EVA01-CLIP text tower of APE-L_A / L_B / L_C (…_lsj1024_cp_12ep.py:83-86).  Same
    constructor keywords plus `tokenizer` (the reference calls OpenAI's `clip.tokenize(texts, context_length=77,
    truncate=True)`, the default here when that package is installed), same `forward_text` dict, parameter names of the
    reference's text half (`net.text.*`, `net.text.logit_scale`).  The weights are read from `cache_dir` (an EVA-CLIP
    checkpoint: `load_eva01_text_state_dict`); a missing or unexpected text entry is an error.  cache_dir=None leaves the
    initialisation (tests, synthetic weights).  dtype "float32" (the reference's default) runs the literal fp32 tower,
    "float16" / "bfloat16" the engine path (wgmma GEMMs, causal flash attention) on CUDA."""

    CONFIGS = {name: dict(embed_dim=1024, text_cfg=dict(context_length=77, vocab_size=49408, width=768, heads=12, layers=12))
               for name in ("EVA_CLIP_g_14", "EVA_CLIP_g_14_X")}  # eva01_clip/model_configs/*.json (text_cfg: identical)

    def __init__(self, clip_model="EVA_CLIP_g_14", cache_dir="eva_clip_psz14.pt", dtype="float32", max_batch_size=2560,
                 tokenizer=None, text_cfg=None, embed_dim=None, pack_prompts=False):
        super().__init__()
        if clip_model not in self.CONFIGS and text_cfg is None:
            raise ValueError(f"ape_b200.EVA01CLIP: unknown clip_model {clip_model!r} (known: {sorted(self.CONFIGS)})")
        cfg = self.CONFIGS.get(clip_model, {})
        self.net = _EVA01Text(text_cfg or cfg["text_cfg"], embed_dim or cfg["embed_dim"])
        if cache_dir is not None:
            sd = load_eva01_text_state_dict(cache_dir)
            missing, unexpected = self.net.text.load_state_dict(sd, strict=False)
            if missing or unexpected:
                raise RuntimeError(f"ape_b200.EVA01CLIP: {cache_dir} does not match the {clip_model} text tower: "
                                   f"missing text.{missing[:4]}, unexpected text.{unexpected[:4]}")
        for p in self.net.parameters():
            p.requires_grad = False
        self._setup(dtype, max_batch_size, tokenizer, pack_prompts)

    def _default_tokenizer(self):
        try:
            from clip import tokenize  # OpenAI CLIP, what clip_wrapper_eva01.py imports
        except Exception as e:  # noqa: BLE001
            raise RuntimeError("ape_b200.EVA01CLIP needs a tokenizer (OpenAI's clip.tokenize) or pre-tokenised int64 [N, 77] "
                               "input") from e
        return lambda texts: tokenize(texts, context_length=77, truncate=True)
