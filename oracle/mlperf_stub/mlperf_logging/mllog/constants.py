def __getattr__(name):      # every constant is its own name
    return name
