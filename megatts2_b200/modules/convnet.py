"""ConvBlock / ConvStack / ResidualBlockStack / ConvNet / ConvNetDoubleLayer / ConvNetDouble
with the reference's surface (modules/convnet.py:9-31, 34-50, 52-72, 74-119, 121-154,
156-210): same ctor kwargs, module tree (hence state_dict keys) and (B, C, T) forward
signatures.  Children hold parameters only; the math runs channels-last in
libmegatts2_b200 (mtts_convnet_forward_f32 / mtts_convnet_double_forward_f32).
``forward_cl`` variants take/return (B, T, C) and skip the two boundary transposes."""
import ctypes as C

import torch
import torch.nn as nn

from .. import _lib as L
from .. import ops, pack


def _act_code(name: str) -> int:
    if name != "ReLU":
        raise L.MttsError(f"activation {name!r} is not on the synthesis path (configs use ReLU)")
    return L.ACT_RELU


class ConvBlock(nn.Module):
    def __init__(self, hidden_size, kernel_size, activation):
        super().__init__()
        self.conv = nn.Conv1d(hidden_size, hidden_size, kernel_size, padding=(kernel_size - 1) // 2)
        self.norm = nn.LayerNorm(hidden_size)
        self.activation = getattr(nn, activation)()
        self.dropout = nn.Dropout(0.1)
        self.kernel_size = kernel_size
        self.act_code = _act_code(activation)

    def forward_cl(self, x, res=None):
        """ReLU -> conv -> LN (convnet.py:22-31), channels-last; `res` is added after the LN
        (fused residual of ResidualBlockStack, convnet.py:71)."""
        if self.training:
            raise L.MttsError("training-mode dropout is outside the synthesis path (call .eval())")
        k = self.kernel_size
        y = ops.conv1d(x, pack.pack_conv(self.conv.weight), self.conv.bias.detach(), k=k, pad=(k - 1) // 2,
                       pre_act=self.act_code)
        return ops.layernorm(y, self.norm.weight.detach(), self.norm.bias.detach(), eps=self.norm.eps, out=y, res=res)

    def forward(self, x):
        return ops.to_channels_first(self.forward_cl(ops.to_channels_last(x)))


class ConvStack(nn.Module):
    def __init__(self, hidden_size, n_blocks, kernel_size, activation):
        super().__init__()
        self.blocks = nn.Sequential(*[ConvBlock(hidden_size, kernel_size, activation) for _ in range(n_blocks)])

    def forward_cl(self, x, res=None):
        n = len(self.blocks)
        for i, b in enumerate(self.blocks):
            x = b.forward_cl(x, res if i == n - 1 else None)
        return x

    def forward(self, x):
        return ops.to_channels_first(self.forward_cl(ops.to_channels_last(x)))


class ResidualBlockStack(nn.Module):
    def __init__(self, hidden_size, n_stacks, n_blocks, kernel_size, activation):
        super().__init__()
        self.conv_stacks = nn.Sequential(
            *[ConvStack(hidden_size, n_blocks, kernel_size, activation) for _ in range(n_stacks)])

    def forward_cl(self, x):
        for cs in self.conv_stacks:
            x = cs.forward_cl(x, res=x)   # x + ConvStack(x): the add is fused into the last LayerNorm
        return x

    def forward(self, x):
        return ops.to_channels_first(self.forward_cl(ops.to_channels_last(x)))


def _run_convnet(struct_ref, ws_fn, fwd_fn, x_cl, t_out, c_out):
    lib = L.lib()
    B, T, _ = x_cl.shape
    y = torch.empty(B, t_out, c_out, dtype=torch.float32, device=x_cl.device)
    ws = ops.workspace(ws_fn(struct_ref, B, T), x_cl.device)
    L.check(fwd_fn(struct_ref, x_cl.data_ptr(), x_cl.stride(0), x_cl.stride(1), y.data_ptr(), y.stride(0), y.stride(1),
                   B, T, ws.data_ptr(), ws.numel(), ops._stream()))
    return y


class ConvNet(pack.PlanMixin, nn.Module):
    def __init__(self, in_channels: int, out_channels: int, hidden_size: int, n_stacks: int, n_blocks: int,
                 kernel_size: int, activation: str, last_layer_avg_pooling: bool = False):
        super().__init__()
        p = (kernel_size - 1) // 2
        self.first_layer = nn.Conv1d(in_channels, hidden_size, kernel_size, stride=1, padding=p)
        self.conv_stack = ResidualBlockStack(hidden_size, n_stacks, n_blocks, kernel_size, activation)
        if last_layer_avg_pooling:
            raise L.MttsError("last_layer_avg_pooling is only used by the (out-of-scope) discriminator")
        self.last_layer = nn.Conv1d(hidden_size, out_channels, kernel_size, stride=1, padding=p)
        self.cfg = (in_channels, out_channels, hidden_size, kernel_size, n_stacks, n_blocks)
        _act_code(activation)
        self._plan = None

    def _plan_get(self):
        engine = getattr(self, "engine", None)
        engine = pack.default_engine() if engine is None else int(engine)
        sig = pack.signature(list(self.parameters())) + (engine,)
        if self._plan is None or self._plan.sig != sig:
            pl = pack.Plan()
            pl.sig = sig
            cin, cout, hid, k, ns, nb = self.cfg
            arr = (L.ConvBlock * (ns * nb))()
            pack.fill_conv_blocks(pl, arr, 0, self.conv_stack, engine)
            pl.hold(arr)
            s = L.ConvNet()
            s.in_channels, s.out_channels, s.hidden, s.k, s.n_stacks, s.n_blocks = cin, cout, hid, k, ns, nb
            s.engine = engine
            s.w_first, s.b_first = pl.p(pack.pack_conv(self.first_layer.weight)), pl.p(self.first_layer.bias)
            s.w_last, s.b_last = pl.p(pack.pack_conv(self.last_layer.weight)), pl.p(self.last_layer.bias)
            s.blocks = C.cast(arr, C.POINTER(L.ConvBlock))
            pl.struct = s
            self._plan = pl
        return self._plan

    def receptive_field(self) -> int:
        """Half-width in frames of what one output frame depends on: first_layer, every ConvBlock and last_layer are
        'same' convolutions of kernel k (20 for k = 5 with 4 x 2 blocks).  A window of frames run on its own gives the
        whole sequence's outputs for the frames at least this far from each window edge that is not a sequence edge."""
        _, _, _, k, ns, nb = self.cfg
        return (k - 1) // 2 * (2 + ns * nb)

    def forward_cl(self, x_cl):
        """(B, T, Cin) -> (B, T, Cout)  (ConvNet.forward, convnet.py:115-119)."""
        if self.training:
            raise L.MttsError("training-mode dropout is outside the synthesis path (call .eval())")
        x_cl = ops._dev(x_cl, name="x")
        if x_cl.stride(2) != 1:
            x_cl = x_cl.contiguous()
        pl = self._plan_get()
        lib = L.lib()
        return _run_convnet(C.byref(pl.struct), lib.mtts_convnet_workspace_bytes, lib.mtts_convnet_forward_f32,
                            x_cl, x_cl.shape[1], self.cfg[1])

    def forward(self, x):
        return ops.to_channels_first(self.forward_cl(ops.to_channels_last(x)))


class ConvNetDoubleLayer(nn.Module):
    def __init__(self, hidden_size: int, n_stacks: int, n_blocks: int, middle_layer: nn.Module, kernel_size: int,
                 activation: str):
        super().__init__()
        self.conv_stack1 = ResidualBlockStack(hidden_size, n_stacks, n_blocks, kernel_size, activation)
        self.middle_layer = middle_layer
        self.conv_stack2 = ResidualBlockStack(hidden_size, n_stacks, n_blocks, kernel_size, activation)

    def forward_cl(self, x):
        x = self.conv_stack1.forward_cl(x)
        x = middle_forward_cl(self.middle_layer, x)
        return self.conv_stack2.forward_cl(x)

    def forward(self, x):
        return ops.to_channels_first(self.forward_cl(ops.to_channels_last(x)))


def _middle_desc(m):
    """(kind, k, stride, pad) of a ConvNetDouble middle layer: MaxPool1d(k, ceil) (vqpe.py:38)
    or a strided Conv1d (mrte.py:101-107)."""
    if isinstance(m, nn.MaxPool1d):
        k = m.kernel_size if isinstance(m.kernel_size, int) else m.kernel_size[0]
        s = m.stride if isinstance(m.stride, int) else m.stride[0]
        if s != k or not m.ceil_mode or m.padding not in (0, (0,)) or m.dilation not in (1, (1,)):
            raise L.MttsError("only MaxPool1d(k, stride=k, ceil_mode=True) is on the synthesis path")
        return 0, k, k, 0
    if isinstance(m, nn.Conv1d):
        if m.dilation[0] != 1 or m.groups != 1 or m.bias is None:
            raise L.MttsError("unsupported middle Conv1d")
        return 1, m.kernel_size[0], m.stride[0], m.padding[0]
    raise L.MttsError(f"unsupported ConvNetDouble middle layer {type(m).__name__}")


def middle_forward_cl(m, x):
    kind, k, s, p = _middle_desc(m)
    if kind == 0:
        return ops.maxpool_time(x, k)
    return ops.conv1d(x, pack.pack_conv(m.weight), m.bias.detach(), k=k, stride=s, pad=p)


class ConvNetDouble(pack.PlanMixin, nn.Module):
    def __init__(self, in_channels: int, out_channels: int, hidden_size: int, n_layers: int, n_stacks: int,
                 n_blocks: int, middle_layer: nn.Module, kernel_size: int, activation: str):
        super().__init__()
        p = (kernel_size - 1) // 2
        self.first_layer = nn.Conv1d(in_channels, hidden_size, kernel_size, stride=1, padding=p)
        # every layer shares the SAME middle_layer module object (convnet.py:182-191): its
        # parameters appear under every layers.{l}.middle_layer.* key, aliasing one storage
        self.layers = nn.Sequential(*[
            ConvNetDoubleLayer(hidden_size, n_stacks, n_blocks, middle_layer, kernel_size, activation)
            for _ in range(n_layers)])
        self.last_layer = nn.Conv1d(hidden_size, out_channels, kernel_size, stride=1, padding=p)
        self.cfg = (in_channels, out_channels, hidden_size, kernel_size, n_layers, n_stacks, n_blocks)
        _act_code(activation)
        self._plan = None

    def _plan_get(self):
        engine = getattr(self, "engine", None)
        engine = pack.default_engine() if engine is None else int(engine)
        sig = pack.signature(list(self.parameters())) + (engine,)
        if self._plan is None or self._plan.sig != sig:
            pl = pack.Plan()
            pl.sig = sig
            cin, cout, hid, k, nl, ns, nb = self.cfg
            arr = (L.ConvBlock * (nl * 2 * ns * nb))()
            i = 0
            for lyr in self.layers:
                i = pack.fill_conv_blocks(pl, arr, i, lyr.conv_stack1, engine)
                i = pack.fill_conv_blocks(pl, arr, i, lyr.conv_stack2, engine)
            pl.hold(arr)
            s = L.ConvNetDouble()
            s.in_channels, s.out_channels, s.hidden, s.k = cin, cout, hid, k
            s.engine = engine
            s.n_layers, s.n_stacks, s.n_blocks = nl, ns, nb
            mid = self.layers[0].middle_layer
            s.middle_kind, s.middle_k, s.middle_stride, s.middle_pad = _middle_desc(mid)
            if s.middle_kind == 1:
                s.w_middle, s.b_middle = pl.p(pack.pack_conv(mid.weight)), pl.p(mid.bias)
            s.w_first, s.b_first = pl.p(pack.pack_conv(self.first_layer.weight)), pl.p(self.first_layer.bias)
            s.w_last, s.b_last = pl.p(pack.pack_conv(self.last_layer.weight)), pl.p(self.last_layer.bias)
            s.blocks = C.cast(arr, C.POINTER(L.ConvBlock))
            pl.struct = s
            self._plan = pl
        return self._plan

    def forward_cl(self, x_cl):
        """(B, T, Cin) -> (B, T_mid, Cout)  (ConvNetDouble.forward, convnet.py:202-210)."""
        if self.training:
            raise L.MttsError("training-mode dropout is outside the synthesis path (call .eval())")
        x_cl = ops._dev(x_cl, name="x")
        if x_cl.stride(2) != 1:
            x_cl = x_cl.contiguous()
        pl = self._plan_get()
        lib = L.lib()
        t_mid = lib.mtts_convnet_double_out_len(C.byref(pl.struct), x_cl.shape[1])
        return _run_convnet(C.byref(pl.struct), lib.mtts_convnet_double_workspace_bytes,
                            lib.mtts_convnet_double_forward_f32, x_cl, t_mid, self.cfg[1])

    def forward(self, x):
        return ops.to_channels_first(self.forward_cl(ops.to_channels_last(x)))
