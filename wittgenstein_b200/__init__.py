"""wittgenstein_b200 — H100-native discrete-event engine behind the Wittgenstein
Protocol / Network / Node / Message surface (hot path only: see DESIGN.md)."""
from ._lib import WtgError  # noqa: F401
from .network import Network  # noqa: F401
from .protocols import (CasperIMD, CasperParemeters, GSFSignature, GSFSignatureParameters, Handel, HandelParameters, P2PFlood,  # noqa: F401
                        P2PFloodParameters, PingPong, PingPongParameters, SanFerminCappos, SanFerminCapposParameters, SanFerminSignature,
                        SanFerminSignatureParameters, Slush, SlushParameters, Snowflake, SnowflakeParameters)
from .run_multiple import (DoneAtStatGetter, MsgReceivedStatGetter, ProgressPerTime, RunMultipleTimes, SimpleStats,  # noqa: F401
                           cont_until_done)
