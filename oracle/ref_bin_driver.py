"""Run the UNMODIFIED reference CLI (dlrm_s_pytorch.run()) on its MLPerf binary-loader path:

    python oracle/ref_bin_driver.py <reference flags>

Two things the reference cannot supply are added from outside: the `mlperf_logging` package (a stub under
oracle/mlperf_stub that writes nothing) and `CriteoBinDataset.num_samples`, which make_criteo_data_and_loaders
reads (dlrm_data_pytorch.py:438) but data_loader_terabyte.CriteoBinDataset does not define."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("DLRM_REFERENCE", "/root/reference")


def main():
    sys.path[:0] = [REF, os.path.join(HERE, "mlperf_stub")]
    import data_loader_terabyte as dlt

    dlt.CriteoBinDataset.num_samples = property(lambda s: os.path.getsize(s.file.name) // (4 * s.tot_fea))
    sys.argv = ["dlrm_s_pytorch.py"] + sys.argv[1:]
    import dlrm_s_pytorch

    dlrm_s_pytorch.run()


if __name__ == "__main__":
    main()
