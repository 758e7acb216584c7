import logging


class _Logger:
    def __init__(self):
        self.logger = logging.getLogger("mllog_stub")

    def start(self, *args, **kwargs):
        pass

    end = event = start


_LOGGER = _Logger()


def get_mllogger():
    return _LOGGER


def config(**kwargs):
    pass
