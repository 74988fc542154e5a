"""BaseNetwork (reference models/networks/base_network.py:5-57) plus the glue that binds a
generator module to its packed CUDA engine."""
import torch.nn as nn
from torch.nn import init


class BaseNetwork(nn.Module):
    NET_ID = None   # 'M' or 'G' for the generators on the CUDA path

    def __init__(self):
        super().__init__()
        self._engine = None
        self._engine_key = None

    @staticmethod
    def modify_commandline_options(parser, is_train):
        return parser

    def print_network(self):
        n = sum(p.numel() for p in self.parameters())
        print("Network [%s] was created. Total number of parameters: %.1f million. "
              "To see the architecture, do print(network)." % (type(self).__name__, n / 1e6))

    def init_weights(self, init_type="normal", gain=0.02):
        """Same rule as the reference (:23-54): only modules whose CLASS NAME contains 'Conv'/'Linear'
        are re-initialised -- gen_conv / gen_deconv are not, so they keep PyTorch's default init."""
        def visit(m):
            cname = type(m).__name__
            if "BatchNorm2d" in cname:
                if getattr(m, "weight", None) is not None:
                    init.normal_(m.weight.data, 1.0, gain)
                if getattr(m, "bias", None) is not None:
                    init.constant_(m.bias.data, 0.0)
            elif hasattr(m, "weight") and ("Conv" in cname or "Linear" in cname):
                if init_type == "normal":
                    init.normal_(m.weight.data, 0.0, gain)
                elif init_type == "xavier":
                    init.xavier_normal_(m.weight.data, gain=gain)
                elif init_type == "xavier_uniform":
                    init.xavier_uniform_(m.weight.data, gain=1.0)
                elif init_type == "kaiming":
                    init.kaiming_normal_(m.weight.data, a=0, mode="fan_in")
                elif init_type == "orthogonal":
                    init.orthogonal_(m.weight.data, gain=gain)
                elif init_type == "none":
                    m.reset_parameters()
                else:
                    raise NotImplementedError("initialization method [%s] is not implemented" % init_type)
                if getattr(m, "bias", None) is not None:
                    init.constant_(m.bias.data, 0.0)
        self.apply(visit)

    # ------------------------------------------------------------------ CUDA engine binding
    def _weights_key(self):
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

    def engine(self):
        """Packed-weights engine for THIS network alone (the other net stays unloaded). Rebuilt when a
        parameter was replaced or modified in place (load_state_dict, .to(), optimiser step)."""
        from sketchedit_b200.engine import Engine
        key = self._weights_key()
        if self._engine is None or key != self._engine_key:
            eng = Engine()
            eng.load_state_dict(self.NET_ID, {k: v for k, v in self.state_dict().items()})
            self._configure_engine(eng)
            eng.finalize()
            self._engine, self._engine_key = eng, key
        return self._engine

    def _configure_engine(self, eng):
        pass
