"""speechbrain.nnet.transducer namespace."""
