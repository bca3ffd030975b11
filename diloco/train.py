"""``python -m diloco.train @configs/1B/h100.toml [--section.key value ...]`` → :func:`prime_b200.train.main`."""

import sys

from prime_b200.train import main, train  # noqa: F401

if __name__ == "__main__":
    main(sys.argv[1:])
