"""Llama-family decode graph over the drop-in operator surface -- the host-side mirror of the reference's module
loop for quantized models (exllamav2/model.py:938-1054 forward_chunk; attn.py:466-638 forward_paged; mlp.py:318-358;
cache.py:306-656 ExLlamaV2Cache_Q4 / _Q6 / _Q8), used by bench.py and the end-to-end tests.

Per decoder layer the call sequence is exactly the reference's:
    cache.get_kv_state (q_to_fp16_kv)  ->  ext_c.q_attn_forward_1  ->  paged attention with kv-append
    ->  cache.store_kv_state (fp16_to_q_kv)  ->  ext_c.q_attn_forward_2  ->  ext_c.q_mlp_forward_
then final RMSNorm + lm_head (gemm_half_q_half).  What differs from the reference is only the host plumbing:
the whole decode step is captured once in ONE CUDA graph (the reference captures per-module graphs after 205 calls,
cuda/graph.cuh:10), positions live in device memory (cache_seqlens) so the graph is replayed unchanged.

Weights are synthetic (exllamav2_b200/synthetic.py): there is no network to fetch checkpoints.
"""
from __future__ import annotations

import ctypes
import math
import os
from dataclasses import dataclass, field

import torch

from . import ext as ext_c
from . import synthetic
from .ext import none_tensor
from .linear import ExLlamaV2Linear

_lib = ext_c.lib
_lib.exl2b_paged_attn_decode.restype = ctypes.c_int
_lib.exl2b_paged_attn_decode.argtypes = [ctypes.c_void_p] * 8 + [ctypes.c_int] * 7 + [ctypes.c_float, ctypes.c_void_p]

PAGE_SIZE = 256       # exllamav2/generator/dynamic.py: page = 256 tokens
# rows of one step (csrc/gemv.cuh): above GEMM_BIG_MIN_ROWS an un-chained stage takes the dense path; a decode step of up to
# DECODE_CHAIN_ROWS sequences runs chained on the 32-row wgmma tile instead (_chains)
GEMM_BIG_MIN_ROWS = 16
DECODE_CHAIN_ROWS = 32


@dataclass
class QuantPlan:
    """EXL2 quantisation recipe per matrix role: (bits, bits_prop, group_size) as conversion/qparams.py QParams."""
    attn: tuple = ((4,), (1.0,), 128)
    mlp: list = field(default_factory=lambda: [((4,), (1.0,), 128)])      # cycled over layers
    head: tuple = ((6,), (1.0,), 128)


@dataclass
class LlamaConfig:
    name: str
    hidden_size: int
    intermediate_size: int
    num_heads: int
    num_kv_heads: int
    head_dim: int
    num_layers: int
    vocab_size: int
    max_seq_len: int = 2048
    norm_eps: float = 1e-5
    rope_theta: float = 10000.0
    plan: QuantPlan = field(default_factory=QuantPlan)


def _mix_4bpw() -> QuantPlan:
    # ~4.0 bpw class with mixed strips (SURVEY.md 8d C3): attn [5,4]@0.1/0.9, MLP 3 of 4 layers [5,4], 1 of 4 [4,3]
    m54 = ((5, 4), (0.1, 0.9), 128)
    m43 = ((4, 3), (0.1, 0.9), 128)
    return QuantPlan(attn=m54, mlp=[m54, m54, m43, m54], head=((6,), (1.0,), 128))


PRESETS = {
    "llama2-7b-4.0bpw": lambda: LlamaConfig("llama2-7b-4.0bpw", 4096, 11008, 32, 32, 128, 32, 32000, plan=_mix_4bpw()),
    "llama2-7b-4bit-g128": lambda: LlamaConfig("llama2-7b-4bit-g128", 4096, 11008, 32, 32, 128, 32, 32000),
    # BASELINE config 4: GPTQ 4-bit, group 128, act-order (q/k/v and gate/up share g_idx)
    "llama2-7b-gptq-g128-act": lambda: LlamaConfig("llama2-7b-gptq-g128-act", 4096, 11008, 32, 32, 128, 32, 32000,
                                                    plan=QuantPlan(attn=("gptq", 128, True), mlp=[("gptq", 128, True)], head=((6,), (1.0,), 128))),
    "tinyllama-1.1b-4.0bpw": lambda: LlamaConfig("tinyllama-1.1b-4.0bpw", 2048, 5632, 32, 4, 64, 22, 32000),
    "llama2-70b-2.5bpw": lambda: LlamaConfig(
        "llama2-70b-2.5bpw", 8192, 28672, 64, 8, 128, 80, 32000,
        plan=QuantPlan(attn=((4, 3), (0.1, 0.9), 128), mlp=[((3, 2), (0.3, 0.7), 64)], head=((6,), (1.0,), 128))),
    # kv width 512: a token's K/V row is exactly one 512-value cache block, so the reference's block-granular re-quantisation
    # (cache.cu:177-184) never touches a neighbouring token and the per-row fused kernel must reproduce its cache bit for bit
    "test-small": lambda: LlamaConfig("test-small", 512, 1408, 8, 8, 64, 2, 512, max_seq_len=512, plan=_mix_4bpw()),
    "test-tiny": lambda: LlamaConfig("test-tiny", 256, 704, 4, 2, 64, 2, 512, max_seq_len=512, plan=_mix_4bpw()),
}


def rope_tables(head_dim: int, max_seq_len: int, base: float, device) -> tuple[torch.Tensor, torch.Tensor]:
    """device.py:118-170 (default RoPE): fp32 tables, then .half()."""
    inv_freq = 1.0 / (base ** (torch.arange(0, head_dim, 2, device=device).float() / head_dim))
    t = torch.arange(max_seq_len, device=device, dtype=torch.float32)
    freqs = torch.einsum("i,j->ij", t, inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.sin().half(), emb.cos().half()


class ExLlamaV2Cache_Q:
    """Quantised K/V cache (cache.py:306-606): uint8 elements + fp16 scales per 32 values, plus ONE shared fp16 temp pair that
    get_kv_state fills for the layer being evaluated (cache.py:464-469).  `wbits` selects the format as in the reference:
    4 = Q4 (4-bit keys and values), 6 = Q6 (8-bit keys, 4-bit values), 8 = Q8 (8-bit keys and values)."""

    wbits = 4

    def __init__(self, cfg: LlamaConfig, batch_size: int, max_seq_len: int, device):
        assert max_seq_len % PAGE_SIZE == 0
        self.cfg, self.device = cfg, device
        self.batch_size, self.max_seq_len = batch_size, max_seq_len
        self.pages = batch_size * max_seq_len // PAGE_SIZE
        kvh, hd = cfg.num_kv_heads, cfg.head_dim
        shp = (self.pages, PAGE_SIZE, kvh, hd)
        wpe_k, wpe_v = ext_c.KV_WEIGHTS_PER_BYTE[self.wbits]          # values per byte, cache.py:66-69
        self.key_states = [torch.zeros(shp[:3] + (hd // wpe_k,), dtype=torch.uint8, device=device) for _ in range(cfg.num_layers)]
        self.value_states = [torch.zeros(shp[:3] + (hd // wpe_v,), dtype=torch.uint8, device=device) for _ in range(cfg.num_layers)]
        self.key_scales = [torch.zeros(shp[:3] + (hd // 32,), dtype=torch.half, device=device) for _ in range(cfg.num_layers)]
        self.value_scales = [torch.zeros_like(self.key_scales[0]) for _ in range(cfg.num_layers)]
        self.temp_k = torch.zeros(shp, dtype=torch.half, device=device)
        self.temp_v = torch.zeros(shp, dtype=torch.half, device=device)
        pps = max_seq_len // PAGE_SIZE
        self.block_table = torch.arange(self.pages, dtype=torch.int32, device=device).view(batch_size, pps)
        self.cache_seqlens = torch.zeros((batch_size,), dtype=torch.int32, device=device)

    def get_kv_state(self, layer: int):
        """cache.py:472-514: dequantise the live part of the layer's cache into the fp16 temp (paged form)."""
        ext_c.q_to_fp16_kv(self.key_states[layer], self.temp_k, self.key_scales[layer],
                           self.value_states[layer], self.temp_v, self.value_scales[layer],
                           self.batch_size, 0, 0, PAGE_SIZE, self.cache_seqlens, self.block_table, self.wbits)
        return self.temp_k, self.temp_v

    def store_kv_state(self, layer: int, q_len: int):
        """cache.py:517-556: quantise the q_len tokens appended at [seqlen, seqlen + q_len)."""
        ext_c.fp16_to_q_kv(self.temp_k, self.key_states[layer], self.key_scales[layer],
                           self.temp_v, self.value_states[layer], self.value_scales[layer],
                           self.batch_size, 0, q_len, PAGE_SIZE, self.cache_seqlens, self.block_table, self.wbits)

    def footprint(self) -> int:
        return sum(t.numel() * t.element_size() for ts in (self.key_states, self.value_states, self.key_scales, self.value_scales) for t in ts)


class ExLlamaV2Cache_Q4(ExLlamaV2Cache_Q):
    wbits = 4


class ExLlamaV2Cache_Q6(ExLlamaV2Cache_Q):
    wbits = 6


class ExLlamaV2Cache_Q8(ExLlamaV2Cache_Q):
    wbits = 8


CACHE_CLASSES = {4: ExLlamaV2Cache_Q4, 6: ExLlamaV2Cache_Q6, 8: ExLlamaV2Cache_Q8}


_FA = [False, None]


def _flash_attn_with_kvcache():
    """flash_attn_with_kvcache if flash-attn imports AND runs on this GPU, else None (probed once)."""
    if not _FA[0]:
        _FA[0] = True
        try:
            from flash_attn import flash_attn_with_kvcache
            dev = torch.device("cuda")
            qq = torch.zeros((1, 1, 1, 64), dtype=torch.half, device=dev)
            kc = torch.zeros((1, 256, 1, 64), dtype=torch.half, device=dev)
            flash_attn_with_kvcache(q=qq, k=qq.clone(), v=qq.clone(), k_cache=kc, v_cache=kc.clone(),
                                    cache_seqlens=torch.zeros((1,), dtype=torch.int32, device=dev),
                                    block_table=torch.zeros((1, 1), dtype=torch.int32, device=dev), causal=True)
            torch.cuda.synchronize()
            _FA[1] = flash_attn_with_kvcache
        except Exception:      # noqa: BLE001
            _FA[1] = None
    return _FA[1]


def _sdpa_prefill(q, k, v, tk, tv, cache, hd):
    """Causal attention of a prompt chunk over the paged fp16 temp cache with torch SDPA (per sequence; identity-free page walk)."""
    B, T, H, _ = q.shape
    KVH = k.shape[2]
    outs = []
    seqlens = cache.cache_seqlens.tolist()
    for b in range(B):
        n0 = int(seqlens[b])
        pages = cache.block_table[b].long()
        kc = tk[pages].reshape(-1, KVH, hd)
        vc = tv[pages].reshape(-1, KVH, hd)
        kc[n0:n0 + T] = k[b]
        vc[n0:n0 + T] = v[b]
        tk[pages] = kc.view(-1, tk.shape[1], KVH, hd)
        tv[pages] = vc.view(-1, tv.shape[1], KVH, hd)
        kk = kc[: n0 + T].transpose(0, 1)
        vv = vc[: n0 + T].transpose(0, 1)
        if H != KVH:
            kk, vv = kk.repeat_interleave(H // KVH, dim=0), vv.repeat_interleave(H // KVH, dim=0)
        mask = torch.ones((T, n0 + T), dtype=torch.bool, device=q.device).tril(diagonal=n0)
        o = torch.nn.functional.scaled_dot_product_attention(q[b].transpose(0, 1), kk, vv, attn_mask=mask)
        outs.append(o.transpose(0, 1))
    return torch.stack(outs)


class _Layer:
    pass


class ExLlamaV2Decoder:
    """Quantized Llama decoder: embedding -> L x (attention block, MLP block) -> norm -> lm_head."""

    def __init__(self, cfg: LlamaConfig, device="cuda:0", seed: int = 0, batch_size: int = 1, cache_len: int | None = None,
                 cache_bits: int = 4):
        if cache_bits not in CACHE_CLASSES:
            raise ValueError(f"cache_bits must be 4 (Q4), 6 (Q6) or 8 (Q8); got {cache_bits}")
        self.cfg, self.device = cfg, torch.device(device)
        dev = self.device
        H, KVH, hd, hid, inter = cfg.num_heads, cfg.num_kv_heads, cfg.head_dim, cfg.hidden_size, cfg.intermediate_size
        gen = torch.Generator(device=dev)
        gen.manual_seed(seed)
        self.weight_bytes = 0          # algorithmic bytes of all linears for one token (SURVEY.md 8d)
        self.layers: list[_Layer] = []
        self.linears: list[ExLlamaV2Linear] = []
        max_rows = max(64, 8 * batch_size)          # rows of one call through the block functions (their temp buffers): 8 tokens per sequence

        def lin(K, N, plan, s, perm_seed=None):
            w = synthetic.random_linear(K, N, plan, device=dev, seed=s, weight_std=1.0 / math.sqrt(K), perm_seed=perm_seed)
            self.weight_bytes += synthetic.algorithmic_bytes(w, 1)
            l = ExLlamaV2Linear(K, N, device=dev)
            l.load(w)
            self.linears.append(l)
            return l

        s = seed * 100003
        for li in range(cfg.num_layers):
            L = _Layer()
            mp = cfg.plan.mlp[li % len(cfg.plan.mlp)]
            # k / v reuse q's row permutation and up reuses gate's, as the reference's converter produces them
            # (conversion/quantize.py:138-139,159: reuse_h copies the activation-order permutation)
            L.q_proj, L.k_proj = lin(hid, H * hd, cfg.plan.attn, s + 1, s + 1), lin(hid, KVH * hd, cfg.plan.attn, s + 2, s + 1)
            L.v_proj, L.o_proj = lin(hid, KVH * hd, cfg.plan.attn, s + 3, s + 1), lin(H * hd, hid, cfg.plan.attn, s + 4)
            L.gate, L.up, L.down = lin(hid, inter, mp, s + 5, s + 5), lin(hid, inter, mp, s + 6, s + 5), lin(inter, hid, mp, s + 7)
            s += 16
            L.input_norm = (1 + 0.1 * torch.randn((hid,), device=dev, generator=gen)).half()
            L.post_norm = (1 + 0.1 * torch.randn((hid,), device=dev, generator=gen)).half()
            L.temp_a = torch.empty((max_rows, inter), dtype=torch.half, device=dev)
            L.temp_b = torch.empty((max_rows, inter), dtype=torch.half, device=dev)
            L.attn = ext_c.make_q_attn(L.input_norm, none_tensor, True, False, cfg.norm_eps, L.q_proj.q_handle, L.k_proj.q_handle,
                                       L.v_proj.q_handle, L.o_proj.q_handle, none_tensor, none_tensor, max_rows, hid, H, KVH, hd,
                                       cfg.max_seq_len, True, 2, hd, none_tensor, none_tensor, none_tensor, none_tensor, False, True)
            L.mlp = ext_c.make_q_mlp(L.post_norm, none_tensor, True, cfg.norm_eps, L.gate.q_handle, L.up.q_handle, L.down.q_handle,
                                     none_tensor, L.temp_a, L.temp_b, none_tensor, max_rows, False, True, none_tensor, none_tensor,
                                     False, True)
            self.layers.append(L)
        self.final_norm = (1 + 0.1 * torch.randn((hid,), device=dev, generator=gen)).half()
        self.lm_head = lin(hid, cfg.vocab_size, cfg.plan.head, s + 9)
        self.embed = (0.02 * torch.randn((cfg.vocab_size, hid), device=dev, generator=gen)).half()
        # one table row per cache position: the fused / stand-alone RoPE kernels index the tables by position and cannot see their length
        cache_len = cache_len or min(cfg.max_seq_len, 1024)
        self.sin, self.cos = rope_tables(hd, max(cfg.max_seq_len, (cache_len + 255) // 256 * 256), cfg.rope_theta, dev)
        self.cache = CACHE_CLASSES[cache_bits](cfg, batch_size, cache_len, dev)
        self.batch_size = batch_size
        # static decode buffers (graph-capturable)
        B = batch_size
        self.ids = torch.zeros((B, 1), dtype=torch.long, device=dev)
        self.x = torch.empty((B, 1, hid), dtype=torch.half, device=dev)
        self.q = torch.empty((B, 1, H * hd), dtype=torch.half, device=dev)
        self.k = torch.empty((B, 1, KVH * hd), dtype=torch.half, device=dev)
        self.v = torch.empty((B, 1, KVH * hd), dtype=torch.half, device=dev)
        self.attn_out = torch.empty((B, 1, H * hd), dtype=torch.half, device=dev)
        self.xn = torch.empty((B, hid), dtype=torch.half, device=dev)
        self.logits = torch.empty((B, cfg.vocab_size), dtype=torch.half, device=dev)
        self.graph = None
        self.pos = 0        # host-side mirror of cache_seqlens (which lives on the device): bounds are checked BEFORE a launch
        # True: attention reads the quantised cache directly (one kernel per layer); False: the reference's sequence
        # q_to_fp16_kv -> attention on the fp16 temp -> fp16_to_q_kv (three kernels + the temp round trip)
        self.fused_attn = os.environ.get("EXL2B_REF_KV_SEQUENCE") is None
        # producer epilogues feed consumer activation buffers (needs the default LAYOUT_TC matrix layout)
        self.chained = os.environ.get("EXL2B_NO_CHAIN") is None
        for L in self.layers:
            L.chain_attn = ext_c.make_chain([L.q_proj.q_handle, L.k_proj.q_handle, L.v_proj.q_handle], L.input_norm)
            L.chain_mlp = ext_c.make_chain([L.gate.q_handle, L.up.q_handle], L.post_norm)
        self.chain_head = ext_c.make_chain([self.lm_head.q_handle], self.final_norm)
        # above one row a chained step runs every matrix on the wgmma kernel, which cannot stage groups of 256+ rows (EXL2 or GPTQ
        # g256+, ungrouped GPTQ; include/exl2_b200.h exl2b_qmatrix_tc_supported)
        self.tc_staged = all(ext_c.qmatrix_tc_supported(l.q_handle) for l in self.linears)
        self.loras: dict[int, list] = {}     # id -> per layer {projection: (A, B)} (load_lora)
        self.lora_ids: list[int] = []         # the active adapters (set_loras)

    LORA_TARGETS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")

    def load_lora(self, rank: int, targets=LORA_TARGETS, scaling: float = 1.0, seed: int = 0) -> int:
        """Register a synthetic adapter of `rank` on the `targets` projections of every layer and return its id (inactive until
        set_loras).  A [in, rank] ~ N(0, 1/in) and B [rank, out] ~ N(0, 0.2^2/rank) * scaling: with the decoder's weights (std
        1/sqrt(in)) the adapter moves each projection's output by about 20 % of its size times `scaling`."""
        bad = set(targets) - set(self.LORA_TARGETS)
        if bad:
            raise ValueError(f"unknown LoRA targets {sorted(bad)}; expected names from {self.LORA_TARGETS}")
        gen = torch.Generator(device=self.device)
        gen.manual_seed(seed)
        layers = []
        for L in self.layers:
            mats = dict(zip(self.LORA_TARGETS, (L.q_proj, L.k_proj, L.v_proj, L.o_proj, L.gate, L.up, L.down)))
            ad = {}
            for t in self.LORA_TARGETS:
                if t not in targets:
                    continue
                K, N = mats[t].in_features, mats[t].out_features
                a = (torch.randn((K, rank), device=self.device, generator=gen) / math.sqrt(K)).half()
                b = (torch.randn((rank, N), device=self.device, generator=gen) * (0.2 * scaling / math.sqrt(rank))).half()
                ad[t] = (a, b)
            layers.append(ad)
        key = id(layers)
        self.loras[key] = layers
        self._register_loras()
        return key

    def unload_lora(self, key: int):
        """Remove an adapter (and deactivate it)."""
        del self.loras[key]
        if key in self.lora_ids:
            self.set_loras([i for i in self.lora_ids if i != key])
        self._register_loras()

    def set_loras(self, ids):
        """Make `ids` (from load_lora) the active adapters of every following step; [] returns to the plain step.  Drops a captured
        graph: capture() again for the new set."""
        unknown = [i for i in ids if i not in self.loras]
        if unknown:
            raise KeyError(f"no adapter loaded under ids {unknown}")
        self.lora_ids = list(ids)
        self.graph = None

    def _register_loras(self):
        """Every loaded adapter on every block handle (the reference's model.update_loras(), lora.py:194)."""
        for li, L in enumerate(self.layers):
            d = {t: ({}, {}) for t in self.LORA_TARGETS}
            for key, layers in self.loras.items():
                for t, (a, b) in layers[li].items():
                    d[t][0][key], d[t][1][key] = a, b
            ext_c.q_attn_set_loras(L.attn, *d["q_proj"], *d["k_proj"], *d["v_proj"], *d["o_proj"])
            ext_c.q_mlp_set_loras(L.mlp, *d["gate_proj"], *d["up_proj"], *d["down_proj"])

    def _chains(self, rows: int, q_len: int = 1) -> bool:
        """Does a step of `rows` rows (batch x new tokens) run the chained schedule?  One row on the integer GEMV always can;
        more rows only when every matrix can be staged by the wgmma kernel (otherwise the blocks take the dense path): up to 8
        rows in any step, and a decode step (one new token per sequence) of 17..32 sequences on the 32-row wgmma tile, which
        reads the packed weights once where the un-chained step reconstructs every matrix.  Above 32 sequences the 64-row tile
        measured slower than the dense path on the 7B preset (DESIGN.md §7), so those steps stay un-chained.  With active
        adapters only one row on the integer GEMV: there each launch leaves its output as a plain row plus a copy for its consumer,
        which forms RMSNorm, RoPE and act·mul itself, so a LoRA launch after it can add the deltas to both (include/exl2_b200.h
        "block forwards").  Above one row the chained launches fuse RoPE, act·mul and the RMSNorm sums into their epilogues, where no
        delta can be added after them, so adapted steps stay on the un-chained block forms."""
        wide = q_len == 1 and GEMM_BIG_MIN_ROWS < rows <= DECODE_CHAIN_ROWS
        if not (self.chained and self.fused_attn and (rows <= 8 or wide)):
            return False
        if self.lora_ids:
            return rows == 1 and self.row_gemv
        return self.tc_staged or (rows == 1 and self.row_gemv)

    @property
    def row_gemv(self) -> bool:
        """Single rows (bs = 1 decode) run on the HBM-bound integer GEMV (csrc/gemv_i8.cu), unless the library was loaded with
        EXL2B_GEMV=tc.  Read from the library, not settable here: a chained single-row launch leaves the head's input in the
        format of the library's path, and a head picked for the other path would read it as garbage."""
        return ext_c.row_gemv_i8()

    # -- one decoder step over `q_len` new tokens per sequence (q_len small; rows = B * q_len) --
    def _forward_tokens(self, x, q, k, v, attn_out, q_len: int):
        cfg, cache = self.cfg, self.cache
        B = self.batch_size
        stream = torch.cuda.current_stream(self.device).cuda_stream
        H, KVH, hd = cfg.num_heads, cfg.num_kv_heads, cfg.head_dim
        if self._chains(B * q_len, q_len):
            return self._forward_tokens_chained(x, q, k, v, attn_out, q_len)
        for li, L in enumerate(self.layers):
            if self.fused_attn and q_len <= 8:
                # past_len = -1: positions come from cache_seqlens on the device (rope.cu:39-43)
                ext_c.q_attn_forward_1(L.attn, x, B, q_len, -1, cache.cache_seqlens, q, k, v, self.sin, self.cos, self.lora_ids)
                ext_c.paged_attn_decode_q4(q.view(B, q_len, H, hd), k.view(B, q_len, KVH, hd), v.view(B, q_len, KVH, hd),
                                           cache.key_states[li], cache.key_scales[li], cache.value_states[li],
                                           cache.value_scales[li], cache.cache_seqlens, cache.block_table,
                                           attn_out.view(B, q_len, H, hd), 1.0 / math.sqrt(hd), wbits=cache.wbits)
                ext_c.q_attn_forward_2(L.attn, x, attn_out, B, q_len, self.lora_ids)
                ext_c.q_mlp_forward_(L.mlp, x, self.lora_ids)
                continue
            tk, tv = cache.get_kv_state(li)
            ext_c.q_attn_forward_1(L.attn, x, B, q_len, -1, cache.cache_seqlens, q, k, v, self.sin, self.cos, self.lora_ids)
            rc = _lib.exl2b_paged_attn_decode(q.data_ptr(), k.data_ptr(), v.data_ptr(), tk.data_ptr(), tv.data_ptr(),
                                              cache.cache_seqlens.data_ptr(), cache.block_table.data_ptr(), attn_out.data_ptr(),
                                              B, q_len, cfg.num_heads, cfg.num_kv_heads, cfg.head_dim, PAGE_SIZE,
                                              cache.block_table.shape[1], 1.0 / math.sqrt(cfg.head_dim), stream)
            if rc:
                raise RuntimeError(_lib.exl2b_last_error().decode())
            cache.store_kv_state(li, q_len)
            ext_c.q_attn_forward_2(L.attn, x, attn_out, B, q_len, self.lora_ids)
            ext_c.q_mlp_forward_(L.mlp, x, self.lora_ids)
        cache.cache_seqlens.add_(q_len)

    def _forward_tokens_chained(self, x, q, k, v, attn_out, q_len: int, head: bool = False, gemv_only: bool = False):
        """Same layer loop with every producer's epilogue feeding its consumer's activation buffer (include/exl2_b200.h
        "chained launches"): 5 launches per layer -- QKV(+norm+rope), attention over the quantised cache, O(+residual),
        gate|up(+norm+act), down(+residual) -- and no stand-alone norm / rope / prep / cache kernels."""
        cfg, cache = self.cfg, self.cache
        B = self.batch_size
        H, KVH, hd = cfg.num_heads, cfg.num_kv_heads, cfg.head_dim
        n = len(self.layers)
        # single rows (the batch-1 integer GEMV): RoPE is left to the attention kernel, which rotates q / k as it reads them
        fuse_rope = self.row_gemv and B * q_len == 1
        for li, L in enumerate(self.layers):
            ext_c.q_attn_forward_1_ex(L.attn, x, B, q_len, -1, cache.cache_seqlens, q, k, v,
                                      None if fuse_rope else self.sin, None if fuse_rope else self.cos, li > 0, self.lora_ids)
            if not gemv_only:        # (bench.py's roofline loop replays exactly the GEMV launches, nothing else)
                ext_c.paged_attn_decode_q4(q.view(B, q_len, H, hd), k.view(B, q_len, KVH, hd), v.view(B, q_len, KVH, hd),
                                           cache.key_states[li], cache.key_scales[li], cache.value_states[li],
                                           cache.value_scales[li], cache.cache_seqlens, cache.block_table,
                                           attn_out.view(B, q_len, H, hd), 1.0 / math.sqrt(hd), L.o_proj.q_handle,
                                           rope=(self.sin, self.cos, 2) if fuse_rope else None, wbits=cache.wbits)
            ext_c.q_attn_forward_2_ex(L.attn, x, attn_out, B, q_len, True, L.chain_mlp, self.lora_ids)
            if li + 1 < n:
                nxt = self.layers[li + 1].chain_attn
            else:
                nxt = self.chain_head if head else None
            ext_c.q_mlp_forward_ex(L.mlp, x, True, nxt, self.lora_ids)
        if not gemv_only:
            cache.cache_seqlens.add_(q_len)

    def _decode_step(self):
        torch.index_select(self.embed, 0, self.ids.view(-1), out=self.x.view(self.batch_size, -1))
        if self.row_gemv and self.batch_size == 1 and self.chained and self.fused_attn:
            self._forward_tokens_chained(self.x, self.q, self.k, self.v, self.attn_out, 1, head=True)
            ext_c.gemv_norm(self.x.view(1, -1), self.lm_head.q_handle, self.final_norm, self.cfg.norm_eps, self.logits, prepared=True)
            return
        if self._chains(self.batch_size):
            self._forward_tokens_chained(self.x, self.q, self.k, self.v, self.attn_out, 1, head=True)
            ext_c.gemm_half_q_half_prepared(self.lm_head.q_handle, self.logits, True, self.cfg.norm_eps)
            return
        self._forward_tokens(self.x, self.q, self.k, self.v, self.attn_out, 1)
        ext_c.rms_norm(self.x.view(self.batch_size, -1), self.final_norm, self.xn, self.cfg.norm_eps)
        ext_c.gemm_half_q_half(self.xn, self.lm_head.q_handle, self.logits, False)

    def capture(self):
        """Capture the whole decode step in one CUDA graph."""
        # the warm-up step and the capture run on a side stream over the decoder's static buffers: everything already queued on the
        # caller's stream (earlier decode steps whose results the caller may not have read yet) has to be finished first
        torch.cuda.synchronize()
        s = torch.cuda.Stream(self.device)
        saved = self.cache.cache_seqlens.clone()
        with torch.cuda.stream(s):
            self._decode_step()                      # warm-up outside capture (lazy workspace allocation)
            torch.cuda.synchronize()
            self.cache.cache_seqlens.copy_(saved)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                self._decode_step()
        torch.cuda.synchronize()
        self.cache.cache_seqlens.copy_(saved)
        self.graph = g

    def decode(self, ids: torch.Tensor) -> torch.Tensor:
        """ids [B, 1] (device) -> logits fp16 [B, vocab]; advances the cache by one token."""
        if self.pos + 1 > self.cache.max_seq_len:
            raise RuntimeError(f"K/V cache is full ({self.pos} of {self.cache.max_seq_len} positions): decode would run past the page table")
        self.pos += 1
        self.ids.copy_(ids)
        if self.graph is not None:
            self.graph.replay()
        else:
            self._decode_step()
        return self.logits

    def prefill(self, ids: torch.Tensor, chunk: int = 8):
        """Feed a prompt [B, T] through the same kernels, `chunk` tokens at a time (keeps every buffer small; the
        prompt is not part of the timed metric)."""
        B, T = ids.shape
        cfg = self.cfg
        H, KVH, hd = cfg.num_heads, cfg.num_kv_heads, cfg.head_dim
        if self.pos + T > self.cache.max_seq_len:
            raise RuntimeError(f"prompt of {T} tokens does not fit the K/V cache ({self.pos} of {self.cache.max_seq_len} positions used)")
        self.pos += T
        for t0 in range(0, T, chunk):
            n = min(chunk, T - t0)
            x = self.embed[ids[:, t0:t0 + n]].contiguous()
            q = torch.empty((B, n, H * hd), dtype=torch.half, device=self.device)
            k = torch.empty((B, n, KVH * hd), dtype=torch.half, device=self.device)
            v = torch.empty_like(k)
            ao = torch.empty_like(q)
            self._forward_tokens(x, q, k, v, ao, n)
        return x

    def prefill_rows(self, ids: torch.Tensor, cache_attn: bool = False):
        """Whole prompt [B, T] in ONE pass per matrix (the many-row path, csrc/gemm_big.cu), in the reference's own op sequence for
        a prompt chunk (attn.py:466-638): get_kv_state -> q_attn_forward_1 -> flash_attn_with_kvcache on the fp16 temp (third-party
        there too; torch SDPA when flash-attn does not run on this GPU) -> store_kv_state -> q_attn_forward_2 -> q_mlp_forward_.

        cache_attn=True: prompt attention straight over the quantised cache instead (csrc/attn_prefill.cu): q_attn_forward_1 ->
        paged_attn_prefill_q, which attends and appends the new rows in one launch -> q_attn_forward_2 -> q_mlp_forward_rows.  No
        fp16 temp, no host synchronisation: the call can be captured in a CUDA graph.  The default stays the reference sequence
        until the two have been measured against each other on the workloads this decoder serves (tools/bench_prefill_attn.py);
        making the new path the default is left to that later decision."""
        if cache_attn:
            return self._prefill_rows_cache_attn(ids)
        B, T = ids.shape
        cfg, cache = self.cfg, self.cache
        H, KVH, hd = cfg.num_heads, cfg.num_kv_heads, cfg.head_dim
        if self.pos + T > cache.max_seq_len:
            raise RuntimeError(f"prompt of {T} tokens does not fit the K/V cache")
        self.pos += T
        x = self.embed[ids].contiguous()
        q = torch.empty((B, T, H * hd), dtype=torch.half, device=self.device)
        k = torch.empty((B, T, KVH * hd), dtype=torch.half, device=self.device)
        v = torch.empty_like(k)
        ta = torch.empty((B * T, cfg.intermediate_size), dtype=torch.half, device=self.device)
        tb = torch.empty_like(ta)
        fa = _flash_attn_with_kvcache()
        for li, L in enumerate(self.layers):
            tk, tv = cache.get_kv_state(li)
            ext_c.q_attn_forward_1(L.attn, x, B, T, -1, cache.cache_seqlens, q, k, v, self.sin, self.cos, self.lora_ids)
            if fa is not None:
                ao = fa(q=q.view(B, T, H, hd), k=k.view(B, T, KVH, hd), v=v.view(B, T, KVH, hd), k_cache=tk, v_cache=tv,
                        cache_seqlens=cache.cache_seqlens, block_table=cache.block_table, causal=True, softmax_scale=1.0 / math.sqrt(hd))
            else:
                ao = _sdpa_prefill(q.view(B, T, H, hd), k.view(B, T, KVH, hd), v.view(B, T, KVH, hd), tk, tv, cache, hd)
            cache.store_kv_state(li, T)
            ext_c.q_attn_forward_2(L.attn, x, ao.reshape(B, T, H * hd), B, T, self.lora_ids)
            ext_c.q_mlp_forward_rows(L.mlp, x.view(B * T, -1), ta, tb, self.lora_ids)
        cache.cache_seqlens.add_(T)
        return x

    def _prefill_rows_cache_attn(self, ids: torch.Tensor):
        B, T = ids.shape
        cfg, cache = self.cfg, self.cache
        H, KVH, hd = cfg.num_heads, cfg.num_kv_heads, cfg.head_dim
        if self.pos + T > cache.max_seq_len:
            raise RuntimeError(f"prompt of {T} tokens does not fit the K/V cache")
        self.pos += T
        x = self.embed[ids].contiguous()
        q = torch.empty((B, T, H * hd), dtype=torch.half, device=self.device)
        k = torch.empty((B, T, KVH * hd), dtype=torch.half, device=self.device)
        v = torch.empty_like(k)
        ao = torch.empty_like(q)
        ta = torch.empty((B * T, cfg.intermediate_size), dtype=torch.half, device=self.device)
        tb = torch.empty_like(ta)
        for li, L in enumerate(self.layers):
            ext_c.q_attn_forward_1(L.attn, x, B, T, -1, cache.cache_seqlens, q, k, v, self.sin, self.cos, self.lora_ids)
            ext_c.paged_attn_prefill_q(q.view(B, T, H, hd), k.view(B, T, KVH, hd), v.view(B, T, KVH, hd), cache.key_states[li],
                                       cache.key_scales[li], cache.value_states[li], cache.value_scales[li], cache.cache_seqlens,
                                       cache.block_table, ao.view(B, T, H, hd), 1.0 / math.sqrt(hd), wbits=cache.wbits)
            ext_c.q_attn_forward_2(L.attn, x, ao, B, T, self.lora_ids)
            ext_c.q_mlp_forward_rows(L.mlp, x.view(B * T, -1), ta, tb, self.lora_ids)
        cache.cache_seqlens.add_(T)
        return x

    def unload(self):
        for L in self.layers:
            ext_c.free_q_attn(L.attn)
            ext_c.free_q_mlp(L.mlp)
        for l in self.linears:
            l.unload()
        self.layers, self.linears = [], []
