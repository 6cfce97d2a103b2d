"""Model-based diffusion as a black-box optimiser (upstream mbd/blackbox): see mbd_opt."""
