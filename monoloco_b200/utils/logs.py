"""utils/logs.py:5-27: a logger that writes INFO records to the console and to a file."""
import logging


def set_logger(log_path):
    """Logger of this module at INFO level, not propagating, with a timestamped handler on `log_path` and a bare
    console handler."""
    logger = logging.getLogger(__name__)
    logger.setLevel(logging.INFO)
    logger.propagate = False
    to_file = logging.FileHandler(log_path)
    to_file.setFormatter(logging.Formatter('%(asctime)s:%(levelname)s: %(message)s'))
    to_console = logging.StreamHandler()
    to_console.setFormatter(logging.Formatter('%(message)s'))
    for handler in (to_file, to_console):
        logger.addHandler(handler)
    return logger
