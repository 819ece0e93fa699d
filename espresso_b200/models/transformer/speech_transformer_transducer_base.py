"""`speech_transformer_transducer_base` (Conformer/Transformer encoder + LSTM prediction network + joint), H100-native.

Mirrors espresso/models/transformer/speech_transformer_transducer_base.py:41-320:
  forward(src_tokens, src_lengths, prev_output_tokens) -> (logits [B, T', U+1, V], encoder_out_lengths)
  joint(enc, dec) = relu(LN(W_e enc)[:, :, None] + LN(W_d dec)[:, None]) -> weight-normalised fc_out (:86-89)
State-dict keys equal the reference's (decoder.embed_tokens, decoder.layers.{i}.weight_ih/.., proj_encoder,
laynorm_proj_encoder, proj_decoder, laynorm_proj_decoder, fc_out.{bias,weight_g,weight_v}).
The prediction network (SpeechLSTMDecoder, espresso/models/speech_lstm.py:766-919: embedding -> dropout_in -> LSTM
layers -> dropout_out) runs on cuDNN through torch, as SURVEY.md §2.1 scopes it; the two projections, LayerNorms,
the joint broadcast, the [B*T'*(U+1), J] x [J, V] output GEMM and the RNN-T loss are espresso_b200 kernels.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import ops as _ops
from ...flat import FlatParams
from ...modules.encoder_engine import LN_EPS, _r8
from ...registry import register_model
from .speech_transformer_config import DEFAULT_MAX_SOURCE_POSITIONS, SpeechTransformerConfig
from .speech_transformer_encoder_model import (ConvBNReLU, SpeechTransformerEncoderForPrediction, _Affine, _Linear,
                                               encoder_inputs)


class _LstmPredictor(nn.Module):
    """Parameter container + cuDNN execution of the reference's LSTMCell stack (keys: embed_tokens.weight,
    layers.{i}.{weight_ih,weight_hh,bias_ih,bias_hh})."""

    def __init__(self, V, embed_dim, hidden, layers, pad, dropout_in, dropout_out):
        super().__init__()
        self.embed_tokens = nn.Embedding(V, embed_dim, padding_idx=pad)
        nn.init.uniform_(self.embed_tokens.weight, -0.1, 0.1)
        nn.init.constant_(self.embed_tokens.weight[pad], 0)
        self.layers = nn.ModuleList([nn.LSTMCell(embed_dim if i == 0 else hidden, hidden) for i in range(layers)])
        for l in self.layers:
            for n, p in l.named_parameters():
                if "weight" in n or "bias" in n:
                    p.data.uniform_(-0.1, 0.1)
        self.hidden, self.dropout_in, self.dropout_out = hidden, dropout_in, dropout_out

    def forward(self, prev_output_tokens):
        x = F.dropout(self.embed_tokens(prev_output_tokens), self.dropout_in, self.training)
        B = x.size(0)
        for l in self.layers:
            h0 = x.new_zeros(1, B, self.hidden)
            w = [l.weight_ih, l.weight_hh, l.bias_ih, l.bias_hh]
            x, _, _ = torch._VF.lstm(x, (h0, h0.clone()), w, True, 1, 0.0, self.training, False, True)
            x = F.dropout(x, self.dropout_out, self.training)
        return x  # [B, U+1, hidden]


class _JointFn(torch.autograd.Function):
    """enc [B,T,d], dec [B,U1,H] -> logits [B,T,U1,ldV]; parameters / their gradients live in the flat buffers."""

    @staticmethod
    def forward(ctx, enc, dec, model):
        B, T, d = enc.shape
        U1, Hd = dec.shape[1], dec.shape[2]
        pe, e0, me, re_ = model.project(enc.reshape(B * T, d), "encoder")
        pd, d0, md, rd = model.project(dec.reshape(B * U1, Hd), "decoder")
        W, g, v, nrm = model.fc_out_weight()
        J = W.shape[1]
        logits, Fj = model.joint_logits(pe.view(B, T, J), pd.view(B, U1, J), W)
        ctx.saved = (enc, dec, e0, me, re_, d0, md, rd, pe, pd, Fj, W, g, v, nrm)
        ctx.model = model
        return logits.view(B, T, U1, -1)

    @staticmethod
    def backward(ctx, dlogits):
        enc, dec, e0, me, re_, d0, md, rd, pe, pd, Fj, W, g, v, nrm = ctx.saved
        fl = ctx.model.flat
        P, G = fl.param, fl.grad
        B, T, d = enc.shape
        U1, Hd = dec.shape[1], dec.shape[2]
        V, J = W.shape
        ldV = _r8(V)
        cells = B * T * U1
        dl = dlogits.reshape(cells, ldV)
        dlv = dl[:, :V] if ldV != V else dl
        dW = torch.zeros(V, J, device=dl.device, dtype=torch.float32)
        _ops.linear_wgrad(dlv, Fj.view(cells, J), dW, G("fc_out.bias"))
        # weight-norm backward
        vn = v / nrm
        dot = (dW * vn).sum(dim=1, keepdim=True)
        G("fc_out.weight_g").add_(dot)
        G("fc_out.weight_v").add_(g / nrm * (dW - dot * vn))
        dF = _ops.linear_dgrad(dlv, W)
        dpe, dpd32 = _ops.joint_bwd(dF.view(B, T, U1, J), Fj)
        de0 = _ops.layer_norm_bwd(dpe.view(B * T, J), e0, me, re_, P("laynorm_proj_encoder.weight"),
                                  G("laynorm_proj_encoder.weight"), G("laynorm_proj_encoder.bias"))
        _ops.linear_wgrad(de0, enc.reshape(B * T, d), G("proj_encoder.weight"), G("proj_encoder.bias"))
        denc = _ops.linear_dgrad(de0, P("proj_encoder.weight")).view(B, T, d)
        dpd = dpd32.to(torch.bfloat16).view(B * U1, J)
        dd0 = _ops.layer_norm_bwd(dpd, d0, md, rd, P("laynorm_proj_decoder.weight"), G("laynorm_proj_decoder.weight"),
                                  G("laynorm_proj_decoder.bias"))
        _ops.linear_wgrad(dd0, dec.reshape(B * U1, Hd).contiguous(), G("proj_decoder.weight"), G("proj_decoder.bias"))
        ddec = _ops.linear_dgrad(dd0, P("proj_decoder.weight")).view(B, U1, Hd)
        return denc, ddec, None


@register_model("speech_transformer_transducer_base", dataclass=SpeechTransformerConfig)
class SpeechTransformerTransducerModelBase(nn.Module):
    def __init__(self, cfg, encoder, decoder, joint_dim):
        super().__init__()
        self.cfg = cfg
        self.encoder, self.decoder = encoder, decoder
        d, Hd = cfg.encoder.embed_dim, decoder.hidden
        V = decoder.embed_tokens.num_embeddings
        self.proj_encoder = _Linear(d, joint_dim, xavier=1.0)
        self.laynorm_proj_encoder = _Affine(joint_dim)
        self.proj_decoder = _Linear(Hd, joint_dim, xavier=1.0)
        self.laynorm_proj_decoder = _Affine(joint_dim)
        fc = nn.utils.weight_norm(nn.Linear(joint_dim, V), name="weight")  # gives bias / weight_g / weight_v
        self.fc_out = nn.Module()
        self.fc_out.bias = nn.Parameter(fc.bias.detach().clone())
        self.fc_out.weight_g = nn.Parameter(fc.weight_g.detach().clone())
        self.fc_out.weight_v = nn.Parameter(fc.weight_v.detach().clone())
        self.num_updates = 0
        self.frontend = None

    @classmethod
    def build_model(cls, cfg, task, decoder_hidden_size=512, decoder_layers=2, decoder_embed_dim=512, joint_dim=512,
                    decoder_dropout_in=0.1, decoder_dropout_out=0.1):
        if cfg.max_source_positions is None:
            cfg.max_source_positions = DEFAULT_MAX_SOURCE_POSITIONS
        e = cfg.encoder
        conv, size = ConvBNReLU.from_config(e.conv_channels, e.conv_kernel_sizes, e.conv_strides, task.feat_dim,
                                            task.feat_in_channels)
        encoder = SpeechTransformerEncoderForPrediction(cfg, pre_encoder=conv, input_size=size, vocab_size=None)
        d_ = task.target_dictionary
        decoder = _LstmPredictor(len(d_), decoder_embed_dim, decoder_hidden_size, decoder_layers, d_.pad(), decoder_dropout_in,
                                 decoder_dropout_out)
        return cls(cfg, encoder, decoder, joint_dim)

    def finalize_(self, device):
        self.to(device)
        flat = FlatParams(self, groups=self.encoder.flat_groups("encoder."), device=device,
                          channels_last=self.encoder.channels_last_params("encoder."))
        self.encoder.finalize_(device, flat=flat, prefix="encoder.")
        return self

    @property
    def flat(self):
        return self.encoder.flat

    def sync_torch_grads_(self):
        """Fold the gradients of the torch-executed parts (conv front, LSTM predictor) into the flat fp32 buffer."""
        self.encoder.sync_torch_grads_()
        self.flat.fold_torch_grads_(self.decoder, "decoder.")

    def set_num_updates(self, n):
        self.num_updates = n
        self.encoder.set_num_updates(n)

    def output_lengths(self, in_lengths):
        return self.encoder.output_lengths(in_lengths)

    # ---- the joint network's pieces, shared by training (_JointFn) and the decoders ------------------------------
    def project(self, x, side):
        """LN(proj_<side>(x)) for side "encoder" or "decoder": x [n, d] -> (out [n, J], and the LayerNorm input, mean and
        rstd its backward reads)."""
        P = self.flat.param
        x0 = _ops.linear(x.contiguous(), P("proj_%s.weight" % side), P("proj_%s.bias" % side))
        y, mean, rstd = _ops.layer_norm_fwd(x0, P("laynorm_proj_%s.weight" % side), P("laynorm_proj_%s.bias" % side), LN_EPS)
        return y, x0, mean, rstd

    def fc_out_weight(self):
        """Weight normalisation of fc_out (nn.utils.weight_norm, dim=0), tiny [V, J] host glue: W = g * v / ||v||_row as
        bf16, with g, v and ||v|| in fp32 for the backward."""
        P = self.flat.param
        g, v = P("fc_out.weight_g").float(), P("fc_out.weight_v").float()
        nrm = v.norm(dim=1, keepdim=True)
        return (g * v / nrm).to(torch.bfloat16).contiguous(), g, v, nrm

    def joint_logits(self, pe, pd, W):
        """pe [B, T, J], pd [B, U1, J], W from fc_out_weight -> (logits bf16 [B*T*U1, ldV], the vocabulary padded to a
        multiple of 8 with zero columns; the joint activations relu(pe[:, :, None] + pd[:, None]) [B, T, U1, J])."""
        (B, T, J), U1, V = pe.shape, pd.shape[1], W.shape[0]
        Fj = _ops.joint_fwd(pe, pd)
        ldV = _r8(V)
        cells = B * T * U1
        logits = torch.zeros(cells, ldV, device=pe.device, dtype=torch.bfloat16) if ldV != V else \
            torch.empty(cells, ldV, device=pe.device, dtype=torch.bfloat16)
        _ops.gemm(Fj.view(cells, J), W, logits, cells, V, J, J, J, ldV, bias=self.flat.param("fc_out.bias"))
        return logits, Fj

    def forward_encoder(self, net_input):
        x, lens, lens_cpu = encoder_inputs(self, net_input["src_tokens"], net_input["src_lengths"],
                                           net_input.get("src_lengths_cpu"))
        return self.encoder(x, lens, src_lengths_cpu=lens_cpu)

    def forward(self, src_tokens, src_lengths, prev_output_tokens, freq_masks=None, time_masks=None, src_lengths_cpu=None,
                time_warp=None, **unused):
        x, lens, lens_cpu = encoder_inputs(self, src_tokens, src_lengths, src_lengths_cpu, freq_masks, time_masks,
                                           time_warp)
        enc = self.encoder(x, lens, src_lengths_cpu=lens_cpu)
        dec = self.decoder(prev_output_tokens)
        logits = _JointFn.apply(enc["b200_out"], dec, self)
        V = self.fc_out.bias.numel()
        self._b200_out = logits
        return logits[..., :V], enc["src_lengths"][0]
