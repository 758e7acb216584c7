"""Stand-in for the `mlperf_logging` package, which the reference's mlperf_logger.py imports: it accepts every
logging call and writes nothing (oracle/ref_bin_driver.py puts it on the path; compliance events are not recorded)."""
