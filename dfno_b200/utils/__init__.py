from .env import *                # noqa: F401,F403
from .misc import *               # noqa: F401,F403
from .timers import *             # noqa: F401,F403
from .checkpoint import *         # noqa: F401,F403
from .gradcheck import *          # noqa: F401,F403
from .debug import *              # noqa: F401,F403
from .logging import *            # noqa: F401,F403
from .optim import *              # noqa: F401,F403
