"""Image conditioner of the image-to-3D cascade (SURVEY.md section 8f row N3) on the library's kernels.

Mirrors the reference's
  sgm.modules.encoders.modules.FrozenDinov2ImageEmbedder   /root/reference/sgm/modules/encoders/modules.py:791-930
  sgm.modules.encoders.modules.PCD_Scaler                  /root/reference/sgm/modules/encoders/modules.py:1746-1768
  sgm.modules.GeneralConditioner (forward, get_unconditional_conditioning)   modules.py:80-195
with the DINOv2 ViT-L/14-reg4 encoder behind the embedder (torch.hub `dinov2_vitl14_reg`, restated at
modules.py:1321-1362) as `Dinov2Encoder`: the image front end and the token assembly are kernels of
dino_ops.cu, every block runs on the DiT's kernels (LayerNorm -> bf16, wgmma GEMMs with bias / head-split /
GELU / fp32 residual-gate epilogues, wgmma flash attention), the final norm on ga_layernorm_rows.  No torch
arithmetic on the encoder path and no CPU fallback.

Precision: bf16 tensor-core operands, fp32 residual stream, fp32 norms and softmax (the reference runs the encoder
under bf16 autocast).  Deliberate deviation: the front end (blur, bicubic resize, normalisation) always runs in fp32,
where the reference computes it in the input image's dtype.

Scope: arch "vitl" at inp_size 518 only (the deployed configs); other sizes need pos_embed interpolation.  No
gradients: the reference freezes the encoder.  Weights never come from the network: pass `state_dict=`, or place the
upstream checkpoint file `dinov2_vitl14_reg4_pretrain.pth` under `torch.hub.get_dir()/checkpoints/`.
"""
import ctypes as C
import os
import re

import torch
import torch.nn as nn

from . import _lib
from . import dit as _dit
from ._lib import GaGemmEpilogue
from .dit import EPI_F32, EPI_GELU_BF16, EPI_HEADS, EPI_RESID_GATE_F32, _p

D, HEADS, N_REG, PATCH, IMG_SIZE = 1024, 16, 4, 14, 518
GRID = IMG_SIZE // PATCH                  # 37
N_PATCH = GRID * GRID                     # 1369
N_TOK = 1 + N_REG + N_PATCH               # 1374: cls | 4 registers | patches
TOK_PITCH = 1408                          # N_TOK rounded up to the attention kernel's 128
K_PITCH = 640                             # 3 * 14 * 14 = 588 im2col columns rounded up to the GEMM's BK = 64
LN_EPS = 1e-6
CHECKPOINT_NAME = "dinov2_vitl14_reg4_pretrain.pth"      # upstream file name of the hub weights


def expected_shapes(depth=24):
    """{key: shape} of the torch.hub dinov2_vitl14_reg state dict (tests/golden/dinov2_vitl14_reg4_keys.json)."""
    s = {"cls_token": (1, 1, D), "register_tokens": (1, N_REG, D), "mask_token": (1, D), "pos_embed": (1, 1 + N_PATCH, D),
         "patch_embed.proj.weight": (D, 3, PATCH, PATCH), "patch_embed.proj.bias": (D,),
         "norm.weight": (D,), "norm.bias": (D,)}
    for i in range(depth):
        p = "blocks.%d." % i
        s.update({p + "norm1.weight": (D,), p + "norm1.bias": (D,), p + "norm2.weight": (D,), p + "norm2.bias": (D,),
                  p + "attn.qkv.weight": (3 * D, D), p + "attn.qkv.bias": (3 * D,),
                  p + "attn.proj.weight": (D, D), p + "attn.proj.bias": (D,),
                  p + "ls1.gamma": (D,), p + "ls2.gamma": (D,),
                  p + "mlp.fc1.weight": (4 * D, D), p + "mlp.fc1.bias": (4 * D,),
                  p + "mlp.fc2.weight": (D, 4 * D), p + "mlp.fc2.bias": (D,)})
    return s


def state_dict_depth(sd):
    ids = {int(m.group(1)) for m in (re.match(r"blocks\.(\d+)\.", k) for k in sd) if m}
    return max(ids) + 1 if ids else 0


def check_state_dict(sd):
    """Strict: the keys must be exactly those of a ViT-L/14-reg4 of the depth the keys state, with its shapes.
    Returns the depth."""
    depth = state_dict_depth(sd)
    want = expected_shapes(depth)
    missing, unexpected = sorted(set(want) - set(sd)), sorted(set(sd) - set(want))
    if missing or unexpected:
        raise RuntimeError("DINOv2 state dict does not match ViT-L/14-reg4 (depth %d): missing keys %s, unexpected keys %s"
                           % (depth, missing, unexpected))
    bad = ["%s %s (want %s)" % (k, tuple(sd[k].shape), want[k]) for k in want if tuple(sd[k].shape) != want[k]]
    if bad:
        raise RuntimeError("DINOv2 state dict: only ViT-L/14 with 4 registers at 518^2 (D = 1024, 16 heads of 64, "
                           "37 x 37 pos_embed) is supported; wrong shapes: %s" % bad)
    if depth == 0:
        raise RuntimeError("DINOv2 state dict has no blocks")
    return depth


def random_state_dict(depth=24, seed=0, device="cpu"):
    """A state dict with the hub layout and random weights that give attention something to do: linear / conv weights
    with std 1/sqrt(fan_in), LayerScale gammas U(0.1, 1), LayerNorm weight 1 + N(0, 0.1) and bias N(0, 0.1), tokens
    and pos_embed N(0, 0.02), other biases N(0, 0.02) except the qkv bias, N(0, 1).  With unit-variance q and k alone
    the logits of a query spread over the keys with std ~1, which leaves attention close to uniform (mean entropy
    ~0.93 ln N on a noise image); the qkv bias doubles the variance of every query, so the spread is ~1.4 and block 0's
    mean entropy drops to ~0.87 ln N.  For tests and benchmarks (there is no network for checkpoints)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shape in expected_shapes(depth).items():
        if k.endswith(".gamma"):
            v = 0.1 + 0.9 * torch.rand(shape, generator=g)
        elif re.search(r"norm\d?\.weight$", k):
            v = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif re.search(r"norm\d?\.bias$", k):
            v = 0.1 * torch.randn(shape, generator=g)
        elif k.endswith(".weight"):
            fan_in = 1
            for n in shape[1:]:
                fan_in *= n
            v = torch.randn(shape, generator=g) / fan_in ** 0.5
        elif k.endswith(".bias"):
            v = (1.0 if k.endswith("qkv.bias") else 0.02) * torch.randn(shape, generator=g)
        else:                                                           # cls / register / mask tokens, pos_embed
            v = 0.02 * torch.randn(shape, generator=g)
        sd[k] = v
    return {k: v.to(device) for k, v in sd.items()}


def default_checkpoint_path():
    return os.path.join(torch.hub.get_dir(), "checkpoints", CHECKPOINT_NAME)


def load_local_checkpoint(path=None):
    """The hub weights from a local file only (never a download).  Raises RuntimeError saying where the file goes."""
    path = path or default_checkpoint_path()
    if not os.path.exists(path):
        raise RuntimeError("DINOv2 weights not found: pass state_dict=, or place the upstream checkpoint %s at %s "
                           "(nothing is downloaded)" % (CHECKPOINT_NAME, path))
    return torch.load(path, map_location="cpu", weights_only=True)


class Dinov2Encoder:
    """DINOv2 ViT-L/14-reg4 forward at 518^2 on libga_b200.so.  `encode(img [B,3,H,W] in [-1,1])` returns
    {"x_norm_clstoken" [B,1024], "x_norm_patchtokens" [B,1369,1024]} (fp32), after the reference embedder's
    preprocess (kornia antialiased bicubic resize to 518, (x+1)/2, ImageNet normalisation)."""
    MAX_GRAPHS = 4                 # captured (B, H, W) kept at a time (oldest dropped first)

    def __init__(self, state_dict, device="cuda:0"):
        self.L = _lib.lib()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("gaussiananything_b200 needs a CUDA device (no CPU fallback)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        sd = state_dict
        self.depth = check_state_dict(sd)
        dev = self.device
        f32 = lambda k: sd[k].detach().to(device=dev, dtype=torch.float32).contiguous()
        b16 = lambda k: sd[k].detach().to(device=dev, dtype=torch.bfloat16).contiguous()
        pw = torch.zeros(D, K_PITCH, device=dev, dtype=torch.float32)
        pw[:, :3 * PATCH * PATCH] = f32("patch_embed.proj.weight").reshape(D, -1)
        self.w = dict(patch_w=pw.to(torch.bfloat16).contiguous(), patch_b=f32("patch_embed.proj.bias"),
                      cls=f32("cls_token").reshape(D), reg=f32("register_tokens").reshape(N_REG, D).contiguous(),
                      pos=f32("pos_embed").reshape(1 + N_PATCH, D).contiguous(),
                      norm_w=f32("norm.weight"), norm_b=f32("norm.bias"))
        self.blocks = []
        for i in range(self.depth):
            p = "blocks.%d." % i
            self.blocks.append(dict(
                n1_w=f32(p + "norm1.weight"), n1_b=f32(p + "norm1.bias"), n2_w=f32(p + "norm2.weight"),
                n2_b=f32(p + "norm2.bias"), qkv_w=b16(p + "attn.qkv.weight"), qkv_b=f32(p + "attn.qkv.bias"),
                proj_w=b16(p + "attn.proj.weight"), proj_b=f32(p + "attn.proj.bias"),
                ls1=f32(p + "ls1.gamma"), ls2=f32(p + "ls2.gamma"),
                w1=b16(p + "mlp.fc1.weight"), b1=f32(p + "mlp.fc1.bias"),
                w2=b16(p + "mlp.fc2.weight"), b2=f32(p + "mlp.fc2.bias")))
        self.use_graph = os.environ.get("GA_B200_DINO_GRAPH", "1") != "0"
        self._graphs = {}                  # (B, H, W) -> (graph, static image, static outputs)

    # ---- launch helpers
    def _gemm(self, A, W, M, N, K, epi, st):
        _lib.check(self.L.ga_gemm_bf16_tn(_p(A), K, _p(W), K, M, N, K, C.byref(epi), _dit._gemm_config(M, N, epi.mode), st),
                   "ga_gemm_bf16_tn")

    @staticmethod
    def _epi(mode, **kw):
        e = GaGemmEpilogue()
        e.mode = mode
        e.eps = LN_EPS
        for k, v in kw.items():
            setattr(e, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
        return e

    def encode(self, img, return_acts=False):
        """img [B, 3, H, W] (CUDA, any float dtype; H, W <= 4096).  The launch sequence is captured once per (B, H, W)
        into a CUDA graph and replayed from a static input buffer; the returned tensors are copies, so they stay valid
        across later calls.  `self.use_graph = False` (or GA_B200_DINO_GRAPH=0) keeps the eager launch sequence.
        return_acts=True (eager) also returns "acts": the residual stream [B, 1374, 1024] after every block."""
        if not img.is_cuda:
            raise RuntimeError("gaussiananything_b200 DINOv2 encoder needs CUDA tensors (no CPU fallback)")
        if img.dim() != 4 or img.shape[1] != 3:
            raise ValueError("expected an image batch [B, 3, H, W], got %s" % (tuple(img.shape),))
        B, _, H, W = img.shape
        dev = self.device
        with torch.cuda.device(dev), torch.no_grad():
            if return_acts or not self.use_graph or torch.cuda.is_current_stream_capturing():
                x = img.to(device=dev, dtype=torch.float32).contiguous()
                out = self._launches(x, [] if return_acts else None)
                return {k: (v.contiguous() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}
            key = (B, H, W)
            slot = self._graphs.get(key)
            if slot is None:
                while len(self._graphs) >= self.MAX_GRAPHS:
                    self._graphs.pop(next(iter(self._graphs)))
                with torch.inference_mode(False):
                    s_img = torch.empty(B, 3, H, W, device=dev, dtype=torch.float32)
                    s_img.copy_(img)
                    self._launches(s_img)                          # warm-up: first-use kernel attributes are set here
                    torch.cuda.synchronize(dev)
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, capture_error_mode="thread_local"):
                        outs = self._launches(s_img)
                slot = self._graphs[key] = (g, s_img, outs)
            g, s_img, outs = slot
            s_img.copy_(img)
            g.replay()
            return {k: v.clone(memory_format=torch.contiguous_format) for k, v in outs.items()}

    def _launches(self, img, acts=None):
        """The launch sequence of one encode on the current stream (eager, or under graph capture)."""
        L, w, dev = self.L, self.w, self.device
        B, _, H, W = img.shape
        R, H16 = B * N_TOK, HEADS
        st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        z = lambda *s, dt=torch.float32: torch.empty(*s, device=dev, dtype=dt)
        bf = torch.bfloat16
        # ---- front end -> patch matrix -> patch-embed GEMM -> token assembly
        nbytes = int(L.ga_dino_frontend_scratch_bytes(B, H, W, IMG_SIZE))
        scratch = z(nbytes, dt=torch.uint8) if nbytes else None
        pm = z(B * N_PATCH, K_PITCH, dt=bf)
        _lib.check(L.ga_dino_frontend(_p(img), B, H, W, IMG_SIZE, PATCH, _p(pm), K_PITCH, _p(scratch), nbytes, st),
                   "ga_dino_frontend")
        pe = z(B * N_PATCH, D)
        self._gemm(pm, w["patch_w"], B * N_PATCH, D, K_PITCH, self._epi(EPI_F32, bias=w["patch_b"], out=pe, ld_out=D), st)
        x = z(R, D)
        _lib.check(L.ga_dino_tokens(_p(pe), _p(w["cls"]), _p(w["reg"]), N_REG, _p(w["pos"]), _p(x), B, N_PATCH, D, st),
                   "ga_dino_tokens")
        # ---- blocks: x += ls1 * proj(attn(norm1(x))); x += ls2 * fc2(gelu(fc1(norm2(x))))
        h, ao, hid = z(R, D, dt=bf), z(R, D, dt=bf), z(R, 4 * D, dt=bf)
        qb = torch.zeros(B * H16, TOK_PITCH, 64, device=dev, dtype=bf)       # padding rows stay finite (zero)
        kb = torch.zeros(B * H16, TOK_PITCH, 64, device=dev, dtype=bf)
        vtb = torch.zeros(B * H16, 64, TOK_PITCH, device=dev, dtype=bf)
        for wb in self.blocks:
            _lib.check(L.ga_layernorm_modulate(_p(x), _p(wb["n1_w"]), _p(wb["n1_b"]), None, None, 0, 1, _p(h), R, D, LN_EPS,
                                               st), "norm1")
            self._gemm(h, wb["qkv_w"], R, 3 * D, D,
                       self._epi(EPI_HEADS, bias=wb["qkv_b"], q=qb, k=kb, vt=vtb, heads=H16, first_part=0,
                                 tok_pitch=TOK_PITCH, rows_per_batch=N_TOK), st)
            _lib.check(L.ga_attention_bf16(_p(qb), _p(kb), _p(vtb), _p(ao), B, H16, N_TOK, N_TOK, TOK_PITCH, TOK_PITCH,
                                           0.125, 0.0, st), "attention")
            # rows_per_batch = R: every row reads the one [D] LayerScale vector as its gate
            self._gemm(ao, wb["proj_w"], R, D, D,
                       self._epi(EPI_RESID_GATE_F32, bias=wb["proj_b"], out=x, ld_out=D, gate=wb["ls1"], gate_ld=D,
                                 rows_per_batch=R), st)
            _lib.check(L.ga_layernorm_modulate(_p(x), _p(wb["n2_w"]), _p(wb["n2_b"]), None, None, 0, 1, _p(h), R, D, LN_EPS,
                                               st), "norm2")
            self._gemm(h, wb["w1"], R, 4 * D, D, self._epi(EPI_GELU_BF16, bias=wb["b1"], out=hid, ld_out=4 * D), st)
            self._gemm(hid, wb["w2"], R, D, 4 * D,
                       self._epi(EPI_RESID_GATE_F32, bias=wb["b2"], out=x, ld_out=D, gate=wb["ls2"], gate_ld=D,
                                 rows_per_batch=R), st)
            if acts is not None:
                acts.append(x.view(B, N_TOK, D).clone())
        y = z(R, D)
        _lib.check(L.ga_layernorm_rows(_p(x), _p(w["norm_w"]), _p(w["norm_b"]), _p(y), R, D, LN_EPS, st), "final norm")
        y = y.view(B, N_TOK, D)
        out = {"x_norm_clstoken": y[:, 0], "x_norm_patchtokens": y[:, 1 + N_REG:]}
        if acts is not None:
            out["acts"] = acts
        return out


def encode_flops(B=1, depth=24):
    """2 x multiply-adds of one encode: the patch-embed GEMM plus per block 24 N D^2 (qkv, proj, fc1, fc2) and
    4 N^2 D (QK^T and PV), N = 1374 tokens, D = 1024 (about 1.02 TFLOP per image at depth 24)."""
    return B * (2 * N_PATCH * 3 * PATCH * PATCH * D + depth * (24 * N_TOK * D * D + 4 * N_TOK * N_TOK * D))


# ---------------------------------------------------------------------------------------------------------------------
# the reference's embedder / conditioner classes (plain torch around the encoder; not on the hot path)
# ---------------------------------------------------------------------------------------------------------------------
class _EmbModel(nn.Module):
    """Attributes of sgm's AbstractEmbModel that GeneralConditioner reads and sets."""

    def __init__(self):
        super().__init__()
        self.is_trainable = False
        self.ucg_rate = 0.0
        self.input_key = None
        self.legacy_ucg_val = None


class FrozenDinov2ImageEmbedder(_EmbModel):
    """Reference constructor arguments; `forward(image, no_dropout=False)` returns (tokens [B,1369,1024],
    z [B,1024]) with output_cls=True, else tokens, both in image.dtype.  Weights: `state_dict=` (hub layout), else
    the local file torch.hub.get_dir()/checkpoints/dinov2_vitl14_reg4_pretrain.pth; nothing is downloaded.
    `encoder=` shares an already built Dinov2Encoder (or any object with the same `encode`)."""

    def __init__(self, arch="vitl", version="dinov2", device="cuda", max_length=77, freeze=True, antialias=True,
                 ucg_rate=0.0, unsqueeze_dim=False, repeat_to_max_len=False, num_image_crops=0, output_tokens=False,
                 output_cls=False, init_device=None, inp_size=224, state_dict=None, encoder=None):
        super().__init__()
        if arch != "vitl" or version != "dinov2":
            raise NotImplementedError("only DINOv2 ViT-L/14-reg4 (arch='vitl') is built; got %s/%s" % (version, arch))
        if inp_size != IMG_SIZE:
            raise NotImplementedError("only inp_size=518 is built (other sizes need pos_embed interpolation); got %s"
                                      % (inp_size,))
        if not antialias:
            raise NotImplementedError("only the antialiased resize (the reference default) is built")
        if encoder is None:
            sd = state_dict if state_dict is not None else load_local_checkpoint()
            encoder = Dinov2Encoder(sd, device)
        self.encoder = encoder
        self.inp_size = inp_size
        self.max_crops = num_image_crops
        self.pad_to_max_len = self.max_crops > 0
        self.repeat_to_max_len = repeat_to_max_len and not self.pad_to_max_len
        self.device = device
        self.max_length = max_length
        self.antialias = antialias
        self.ucg_rate = ucg_rate
        self.unsqueeze_dim = unsqueeze_dim
        self.output_tokens = output_tokens
        self.output_cls = output_cls

    def freeze(self):
        return self.eval()

    def encode_with_vision_transformer(self, img):
        if img.dim() == 5:
            img = img.flatten(0, 1)                         # b n c h w -> (b n) c h w
        out = self.encoder.encode(img)
        if not self.output_cls:
            return out["x_norm_patchtokens"]
        return out["x_norm_clstoken"], out["x_norm_patchtokens"]

    def forward(self, image, no_dropout=False, **kwargs):
        tokens = self.encode_with_vision_transformer(image)
        z = None
        if self.output_cls:
            z, tokens = tokens
            z = z.to(image.dtype)
        tokens = tokens.to(image.dtype)
        if self.ucg_rate > 0.0 and not no_dropout and not (self.max_crops > 0):
            keep = lambda t: torch.bernoulli((1.0 - self.ucg_rate) * torch.ones(t.shape[0], device=t.device))
            if z is not None:
                z = keep(z)[:, None] * z
            tokens = keep(tokens)[:, None, None] * tokens
        if self.output_cls:
            return tokens, z
        return tokens

    def encode(self, image):
        return self(image)


class PCD_Scaler(_EmbModel):
    """pcd / scaling_factor (optionally perturbed and clipped first, as the reference does)."""

    def __init__(self, scaling_factor=0.45, perturb_pcd_scale=0.0):
        super().__init__()
        self.scaling_factor = scaling_factor
        self.perturb_pcd_scale = perturb_pcd_scale

    def forward(self, pcd, **kwargs):
        if self.perturb_pcd_scale > 0:
            t = torch.rand(pcd.shape[0], 1, 1).to(pcd) * self.perturb_pcd_scale
            pcd = (pcd + t * torch.randn_like(pcd)).clip(-0.45, 0.45)
        return pcd / self.scaling_factor


_EMBEDDERS = {"FrozenDinov2ImageEmbedder": FrozenDinov2ImageEmbedder, "PCD_Scaler": PCD_Scaler}


def _instantiate(cfg):
    name = str(cfg["target"]).rsplit(".", 1)[-1]
    if name not in _EMBEDDERS:
        raise NotImplementedError("embedder %s is not built here (only %s)" % (cfg["target"], sorted(_EMBEDDERS)))
    return _EMBEDDERS[name](**dict(cfg.get("params", None) or {}))


class GeneralConditioner(nn.Module):
    """The part of sgm's GeneralConditioner the image-to-3D sampler uses.  `emb_models`: embedder configs
    ({"target", "params", "input_key", "ucg_rate", "is_trainable", "legacy_ucg_value"}) or embedder modules.
    Output keys: an embedder whose input_key is 'img' or 'caption' maps an output of dimension d to
    '<input_key>_<vector|crossattn|concat>'; any other 3-D output with 3 channels is 'fps-xyz'."""
    OUTPUT_DIM2KEYS = {2: "vector", 3: "crossattn", 4: "concat", 5: "concat"}
    KEY2CATDIM = {"vector": 1, "crossattn": 2, "concat": 1}

    def __init__(self, emb_models):
        super().__init__()
        embedders = []
        for cfg in emb_models:
            if isinstance(cfg, nn.Module):
                embedders.append(cfg)
                continue
            e = _instantiate(cfg)
            e.is_trainable = cfg.get("is_trainable", False)
            e.ucg_rate = cfg.get("ucg_rate", 0.0)
            if "input_key" in cfg:
                e.input_key = cfg["input_key"]
            elif "input_keys" in cfg:
                e.input_keys = cfg["input_keys"]
            else:
                raise KeyError("need either 'input_key' or 'input_keys' for embedder %s" % type(e).__name__)
            e.legacy_ucg_val = cfg.get("legacy_ucg_value", None)
            if e.legacy_ucg_val is not None:
                import numpy as np
                e.ucg_prng = np.random.RandomState()
            embedders.append(e)
        for e in embedders:
            if not getattr(e, "is_trainable", False):
                for prm in e.parameters():
                    prm.requires_grad = False
                e.eval()
        self.embedders = nn.ModuleList(embedders)

    def possibly_get_ucg_val(self, embedder, batch):
        p, val = embedder.ucg_rate, embedder.legacy_ucg_val
        for i in range(len(batch[embedder.input_key])):
            if embedder.ucg_prng.choice(2, p=[1 - p, p]):
                batch[embedder.input_key][i] = val
        return batch

    def _embed(self, batch):
        """[(embedder, [outputs])]: every embedder run once."""
        raw = []
        for e in self.embedders:
            with torch.no_grad():
                if getattr(e, "input_key", None) is not None:
                    if getattr(e, "legacy_ucg_val", None) is not None:
                        batch = self.possibly_get_ucg_val(e, batch)
                    out = e(batch[e.input_key])
                else:
                    out = e(*[batch[k] for k in e.input_keys])
            assert isinstance(out, (torch.Tensor, list, tuple)), \
                "encoder outputs must be tensors or a sequence, but got %s" % type(out)
            raw.append((e, list(out) if isinstance(out, (list, tuple)) else [out]))
        return raw

    def _assemble(self, raw, force_zero_embeddings):
        output = {}
        force_zero_embeddings = force_zero_embeddings or []
        for e, outs in raw:
            key_in = getattr(e, "input_key", None)
            for emb in outs:
                if key_in in ("caption", "img"):
                    out_key = "%s_%s" % (key_in, self.OUTPUT_DIM2KEYS[emb.dim()])
                elif emb.dim() == 3 and emb.shape[-1] == 3:
                    out_key = "fps-xyz"
                else:
                    out_key = self.OUTPUT_DIM2KEYS[emb.dim()]
                if e.ucg_rate > 0.0 and getattr(e, "legacy_ucg_val", None) is None:
                    keep = torch.bernoulli((1.0 - e.ucg_rate) * torch.ones(emb.shape[0], device=emb.device))
                    emb = keep.view(-1, *([1] * (emb.dim() - 1))) * emb
                if key_in is not None and key_in in force_zero_embeddings:
                    emb = torch.zeros_like(emb)
                if out_key in output:
                    output[out_key] = torch.cat((output[out_key], emb), self.KEY2CATDIM[out_key.split("_")[1]])
                else:
                    output[out_key] = emb
        return output

    def forward(self, batch, force_zero_embeddings=None):
        return self._assemble(self._embed(batch), force_zero_embeddings)

    def get_unconditional_conditioning(self, batch_c, batch_uc=None, force_uc_zero_embeddings=None,
                                       force_cond_zero_embeddings=None):
        """(c, uc) with every ucg_rate forced to 0.  With batch_uc None the embedders run once and uc is assembled
        from the same outputs (the reference runs them twice; with dropout off they are deterministic, so the result
        is the same)."""
        rates = [e.ucg_rate for e in self.embedders]
        for e in self.embedders:
            e.ucg_rate = 0.0
        try:
            raw_c = self._embed(batch_c)
            c = self._assemble(raw_c, force_cond_zero_embeddings)
            uc = self._assemble(raw_c if batch_uc is None else self._embed(batch_uc), force_uc_zero_embeddings)
        finally:
            for e, r in zip(self.embedders, rates):
                e.ucg_rate = r
        return c, uc
