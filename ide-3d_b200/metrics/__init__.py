"""Quality metrics of the reference's metrics/ package: FID, KID, precision / recall and IS (metric_main.calc_metric)."""
