"""Top-level drop-in so the reference drivers' `from tokenflow_utils import *`
(run_tokenflow_pnp.py:16, run_tokenflow_sdedit.py:15) resolves to the H100 hook layer."""
from tokenflow_b200.tokenflow_utils import *  # noqa: F401,F403
from tokenflow_b200.tokenflow_utils import __all__  # noqa: F401
