"""MRTE / LengthRegulator with the reference's surface (modules/mrte.py:34-60, 63-183): same
ctor kwargs, attributes (.hidden_size .mel_bins .n_heads), state_dict keys (incl. the shared
strided conv appearing as ``mel_encoder_middle_layer.*`` and ``mel_encoder.layers.{l}.middle_layer.*``)
and method signatures.  ``tc_latent`` additionally accepts the 3-argument form the reference's
own (broken) callers use (mrte.py:180, models/megatts2.py:83)."""
import torch
import torch.nn as nn

from .. import _lib as L
from .. import ops
from .. import sampling as S
from .convnet import ConvNetDouble
from .embedding import SinePositionalEmbedding, TokenEmbedding
from .tokenizer import HIFIGAN_HOP_LENGTH, HIFIGAN_MEL_CHANNELS, HIFIGAN_SR
from .transformer import MultiHeadAttention, TransformerEncoder, TransformerEncoderLayer


class LengthRegulator(nn.Module):
    """Length Regulator from FastSpeech (mrte.py:34-60) as a device-side gather."""

    def __init__(self, mel_frames, sample_rate, duration_token_ms):
        super().__init__()
        assert (mel_frames / sample_rate * 1000 / duration_token_ms) == 1

    def forward(self, x: torch.Tensor, duration_tokens: torch.Tensor, mel_max_length=None):
        """x (B,T,D), duration_tokens (B,T) int -> (B, max_b sum(d_b) [or mel_max_length], D)."""
        d = duration_tokens.to(device=x.device, dtype=torch.int32)
        y, _ = ops.length_regulate(x, d, l_out=None)
        if mel_max_length:
            pad = mel_max_length - y.size(1)
            assert pad >= 0
            if pad:
                z = torch.zeros(y.size(0), mel_max_length, y.size(2), dtype=y.dtype, device=y.device)
                z[:, :y.size(1)] = y
                y = z
        return y


def check_prompts(mels, B, mel_bins, name, device):
    """Every prompt of the list ``mels`` is a CUDA fp32 (B, Tm >= 1, mel_bins) tensor on ``device``."""
    for k, m in enumerate(mels):
        ops._dev(m, name=f"{name}[{k}]")
        if m.dim() != 3 or m.shape[0] != B or m.shape[2] != mel_bins or m.shape[1] < 1:
            raise L.MttsError(f"{name}[{k}]: expected ({B}, Tm, {mel_bins}), got {tuple(m.shape)}")
        if m.device != device:
            raise L.MttsError(f"{name}[{k}]: on {m.device}, expected {device}")


class MRTE(nn.Module):
    def __init__(self, mel_bins: int = HIFIGAN_MEL_CHANNELS, mel_frames: int = HIFIGAN_HOP_LENGTH,
                 mel_activation: str = 'ReLU', mel_kernel_size: int = 3, mel_stride: int = 16, mel_n_layer: int = 5,
                 mel_n_stack: int = 5, mel_n_block: int = 2, content_ff_dim: int = 1024, content_n_heads: int = 2,
                 content_n_layers: int = 8, hidden_size: int = 512,
                 duration_token_ms: float = (HIFIGAN_HOP_LENGTH / HIFIGAN_SR * 1000), phone_vocab_size: int = 320,
                 dropout: float = 0.1, sample_rate: int = HIFIGAN_SR):
        super().__init__()
        self.n_heads = content_n_heads
        self.mel_bins = mel_bins
        self.hidden_size = hidden_size
        self.phone_embedding = TokenEmbedding(dim_model=hidden_size, vocab_size=phone_vocab_size, dropout=dropout)
        self.phone_pos_embedding = SinePositionalEmbedding(dim_model=hidden_size, dropout=dropout)
        self.mel_encoder_middle_layer = nn.Conv1d(hidden_size, hidden_size, kernel_size=mel_stride + 1,
                                                  stride=mel_stride, padding=mel_stride // 2)
        self.mel_encoder = ConvNetDouble(
            in_channels=mel_bins, out_channels=hidden_size, hidden_size=hidden_size, n_layers=mel_n_layer,
            n_stacks=mel_n_stack, n_blocks=mel_n_block, middle_layer=self.mel_encoder_middle_layer,
            kernel_size=mel_kernel_size, activation=mel_activation)
        self.phone_encoder = TransformerEncoder(
            TransformerEncoderLayer(dim=hidden_size, ff_dim=content_ff_dim, conv_ff=True, n_heads=content_n_heads,
                                    dropout=dropout),
            num_layers=content_n_layers)
        self.mha = MultiHeadAttention(qkv_dim=hidden_size, n_heads=1, dropout=dropout)
        self.norm = nn.LayerNorm(hidden_size)
        self.activation = nn.ReLU()
        self.length_regulator = LengthRegulator(mel_frames, sample_rate, duration_token_ms)

    def encode_prompt(self, mel: torch.Tensor) -> torch.Tensor:
        """The mel encoder's output for a prompt mel (B, Tm, mel_bins) -> (B, ceil(Tm / 16), hidden) channels-last: what
        ``tc_latent`` attends to.  Passing it back as ``mel_context=`` gives the same latent bit for bit without encoding
        the prompt again (long-form synthesis encodes its prompt once per passage)."""
        if self.training:
            raise L.MttsError("training-mode dropout is outside the synthesis path (call .eval())")
        return self.mel_encoder.forward_cl(mel)

    def tc_latent(self, phone: torch.Tensor, *args, mel_context: torch.Tensor = None):
        """tc_latent(phone (B,Tp) int64, mel (B,Tm,mel_bins)) -> (B,Tp,hidden), >= 0  (mrte.py:154-171).
        Also accepts tc_latent(phone, phone_lens, mel): phone_lens is ignored, exactly like the
        unmasked reference computation.  ``mel_context``: ``encode_prompt(mel)``, computed earlier; the mel argument
        is then not read."""
        mel = args[-1] if args else None
        if self.training:
            raise L.MttsError("training-mode dropout is outside the synthesis path (call .eval())")
        pe = self.phone_pos_embedding
        pe.extend_pe(phone)
        # embedding gather + alpha * sine PE in one kernel (mrte.py:159-160)
        x = ops.embed_pe(phone, self.phone_embedding.word_embeddings.weight.detach(), pe.pe, pe.alpha_host())
        if mel_context is None:
            mel_context = self.mel_encoder.forward_cl(mel)         # (B, Tm/16, H), already channels-last
        phone_x = self.phone_encoder(x)
        y = self.mha(phone_x, kv=mel_context)
        # LayerNorm -> ReLU fused (mrte.py:168-169)
        return ops.layernorm(y, self.norm.weight.detach(), self.norm.bias.detach(), eps=self.norm.eps,
                             post_act=L.ACT_RELU, out=y)

    def attend(self, phone: torch.Tensor, mels, mel_context=None) -> torch.Tensor:
        """The pre-norm attention outputs of K mels: phone (B,Tp) int64, ``mels`` K tensors (B, Tm_k, mel_bins) ->
        ys (K, B, Tp, hidden), ys[k] = MHA(phone_x, kv=mel_encoder(mels[k])), the y of ``tc_latent(phone, mels[k])`` bit
        for bit.  The phone encoder runs once; each mel runs its mel encoder and the MHA.  ``mel_context``: a list of K
        entries, each ``encode_prompt(mels[k])`` or None; a given entry replaces that mel's encoder pass."""
        if self.training:
            raise L.MttsError("training-mode dropout is outside the synthesis path (call .eval())")
        pe = self.phone_pos_embedding
        pe.extend_pe(phone)
        x = ops.embed_pe(phone, self.phone_embedding.word_embeddings.weight.detach(), pe.pe, pe.alpha_host())
        phone_x = self.phone_encoder(x)
        ys = torch.empty(len(mels), *phone_x.shape, dtype=torch.float32, device=phone_x.device)
        for k, mel in enumerate(mels):
            ctx = None if mel_context is None else mel_context[k]
            self.mha(phone_x, kv=self.mel_encoder.forward_cl(mel) if ctx is None else ctx, out=ys[k])
        return ys

    def norm_relu(self, y: torch.Tensor) -> torch.Tensor:
        """ReLU(LayerNorm(y)) into a new tensor: ``tc_latent``'s last step (mrte.py:168-169)."""
        return ops.layernorm(y, self.norm.weight.detach(), self.norm.bias.detach(), eps=self.norm.eps,
                             post_act=L.ACT_RELU)

    def norm_relu_mix(self, ys: torch.Tensor, weights: torch.Tensor) -> torch.Tensor:
        """ReLU(LayerNorm(sum_k w^_k ys[k])) (ops.mix_layernorm) for the validated CPU ``weights`` (B, K) or (B, Tp, K)."""
        return ops.mix_layernorm(ys, weights.to(ys.device), self.norm.weight.detach(), self.norm.bias.detach(),
                                 eps=self.norm.eps, post_act=L.ACT_RELU)

    def tc_latent_mix(self, phone: torch.Tensor, mels, weights) -> torch.Tensor:
        """Timbre interpolation: the MRTE latent of a weighted mix of K prompts.  ``mels``: K tensors (B, Tm_k, mel_bins)
        (the Tm_k may differ); ``weights``: (K,), (B, K) or (B, Tp, K) with one row per phone, >= 0, each row with a
        positive sum (normalised to w^).  -> (B, Tp, hidden) = ReLU(LayerNorm(sum_k w^_k y_k)), y_k the pre-norm attention
        output of ``tc_latent(phone, mels[k])``: since the out-projection is affine, that is attention under the
        w^-weighted mixture of the per-prompt attention distributions, normalised back onto the latent's scale.  A row
        with one positive weight, on source k, is ``tc_latent(phone, mels[k])``'s row bit for bit.  The phone encoder
        runs once (``attend``); include/megatts2_b200.h (mtts_mix_layernorm_f32) states the mix."""
        if isinstance(mels, torch.Tensor) or not len(mels):
            raise L.MttsError("tc_latent_mix: mels must be a non-empty list of (B, Tm, mel_bins) tensors")
        if phone.dim() != 2:
            raise L.MttsError(f"tc_latent_mix: phone must be (B, Tp), got {tuple(phone.shape)}")
        B, Tp = phone.shape
        w = S.synth_mix_weights(weights, len(mels), B, Tp, "tc_latent_mix weights")
        check_prompts(mels, B, self.mel_bins, "mels", phone.device)
        return self.norm_relu_mix(self.attend(phone, mels), w)

    def forward(self, duration_tokens: torch.Tensor, phone: torch.Tensor, phone_lens: torch.Tensor,
                mel: torch.Tensor):
        tc = self.tc_latent(phone, phone_lens, mel)
        return self.length_regulator(tc, duration_tokens)
