// Hand-written source: go/generate.py derives the bls12-377, bls12-381 and bw6-761 packages from this file.

//go:build !b200

package bn254

import (
	"io"

	"github.com/consensys/gnark/backend/groth16/bn254/mpcsetup"
)

const noTag = "b200 backend requested but program compiled without 'b200' build tag"

// ContributePhase2 is the b200 build's (see there).
func ContributePhase2(p *mpcsetup.Phase2) error { panic(noTag) }

// ContributePhase1 is the b200 build's (see there).
func ContributePhase1(r io.Reader, w io.Writer) error { panic(noTag) }
