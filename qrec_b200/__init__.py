"""qrec_b200: H100-native engine behind QRec's BPR / LightGCN / NeuMF hot path (see README.md)."""
